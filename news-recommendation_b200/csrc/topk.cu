// Top-k recommendation over a whole news pool (include/newsrec_b200.h, nr_topk_dot): score[u][n] = users[u] . news[n] for
// every user and news at fp32 level on the tensor cores, and only the k best news of each user leave the kernel.
//
// Operands: users and news are split into hi/lo bf16 planes (rows_to_bf16, one launch) and every score is
//   hi_u . hi_n + hi_u . lo_n + lo_u . hi_n      (three m64n64k16 wgmmas per k-step into one fp32 accumulator)
// hi + lo carries x to ~2^-17 relative, so the dropped lo . lo term and the plane roundings leave at most
// 2^-15 sum_i |u_i||n_i| of the fp32 dot product, and the tensor-core fp32 accumulation of 3 round_up(D, 64) products adds
// at most 3 round_up(D, 64) 2^-23 sum_i |u_i||n_i|:  |score - u.n| <= (2^-15 + 3 round_up(D, 64) 2^-23) sum_i |u_i||n_i|.
//
// Decomposition: CTA (m, s) owns 64 users (tile m) and the news tiles of split s.  A TMA producer warp streams, per news tile
// of 64 rows and per 64-column k-chunk, the users' hi/lo boxes and the news' hi/lo boxes (32 KB) through a 3-stage mbarrier
// ring; one consumer warpgroup issues the wgmmas.  The 64 x 64 score tile stays in the accumulator fragments: a score enters
// its user's candidate buffer in shared memory (256 entries) only if it beats the user's threshold, the k-th best score of the
// buffer's last merge (-inf before).  A buffer that could not take another tile is merged: one warp sorts it by (score
// descending, news row ascending) and keeps the k best.  Later tiles hold higher rows, so a score equal to the threshold
// never displaces it: "beats" is a strict >, and equal scores keep the lower row.  The matrix of scores never reaches
// memory; per (user, split) k (score, row) pairs do, and with several splits one small kernel merges them.
#include <algorithm>
#include <cmath>

#define NR_WATCHDOG_SYMBOL g_topk_dev_error
#include "nr_fused.cuh"
#include "nr_ops.h"

namespace nr {

int read_topk_device_error(int* out4) {
    return static_cast<int>(cudaMemcpyFromSymbol(out4, fused::g_topk_dev_error, sizeof(int) * 4));
}

namespace topk {

using namespace fused;

constexpr int kUsers = 64;                  // users per CTA (wgmma M)
constexpr int kNews = 64;                   // news per tile (wgmma N)
constexpr int kBox = 64 * 128;              // one 64-row x 64-column bf16 box, 128-byte swizzled
constexpr int kStage = 4 * kBox;            // users hi | users lo | news hi | news lo
constexpr int kStages = 3;
constexpr int kCap = 256;                   // candidate buffer per user: k <= 128 after a merge + the survivors of 2 tiles
constexpr int kThreads = 5 * 32;            // one consumer warpgroup + the TMA producer warp
constexpr int kMaxSplits = 8;
constexpr size_t kSmem = 1024 + kStages * kStage + kUsers * kCap * 8 + 1024;
static_assert(kSmem <= 232448, "topk_dot_kernel: shared memory");

struct Params {
    long long n_users;
    int n_news, k, k_chunks, tiles, splits;
    const long long* excl_offsets;  // [n_users + 1] or null
    const long long* excl_rows;
    long long* idx;                 // splits == 1: [n_users][k]
    float* score;
    float* part_score;              // splits > 1: [n_users][splits][k]
    int* part_row;
    int* bad_row_flag;
    int* bad_score_flag;
};

// a before b in the output order: higher score, then lower row
__device__ __forceinline__ bool before(float sa, int ra, float sb, int rb) { return sa > sb || (sa == sb && ra < rb); }

// one warp sorts n (a power of two, <= 1024) (score, row) pairs in shared memory into output order (bitonic)
__device__ void warp_sort(float* s, int* r, int n) {
    const int lane = threadIdx.x & 31;
    for (int size = 2; size <= n; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = lane; i < n / 2; i += 32) {
                const int a = 2 * i - (i & (stride - 1)), b = a + stride;
                const bool up = (a & size) == 0;
                const float sa = s[a], sb = s[b];
                const int ra = r[a], rb = r[b];
                if (up ? before(sb, rb, sa, ra) : before(sa, ra, sb, rb)) {
                    s[a] = sb; s[b] = sa;
                    r[a] = rb; r[b] = ra;
                }
            }
            __syncwarp();
        }
}

// sorts user buffer u (pads [cnt, kCap) with (-inf, INT_MAX)), keeps the k best, sets the threshold
__device__ void merge_user(float* bs, int* br, int* cnt, float* thr, int u, int k) {
    const int lane = threadIdx.x & 31;
    float* s = bs + u * kCap;
    int* r = br + u * kCap;
    const int c = cnt[u];
    for (int i = c + lane; i < kCap; i += 32) {
        s[i] = -INFINITY;
        r[i] = 0x7fffffff;
    }
    __syncwarp();
    warp_sort(s, r, kCap);
    if (lane == 0) {
        cnt[u] = min(c, k);
        thr[u] = c >= k ? s[k - 1] : -INFINITY;
    }
    __syncwarp();
}

__global__ void __launch_bounds__(kThreads, 1) topk_dot_kernel(const __grid_constant__ CUtensorMap tmUh, const __grid_constant__ CUtensorMap tmUl,
                                                               const __grid_constant__ CUtensorMap tmNh, const __grid_constant__ CUtensorMap tmNl,
                                                               const Params p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sStage = base;
    float* bs = reinterpret_cast<float*>(sStage + kStages * kStage);   // [kUsers][kCap] candidate scores
    int* br = reinterpret_cast<int*>(bs + kUsers * kCap);               // [kUsers][kCap] candidate rows
    uint64_t* full = reinterpret_cast<uint64_t*>(br + kUsers * kCap);   // [kStages]
    uint64_t* empty = full + kStages;                                   // [kStages]
    int* cnt = reinterpret_cast<int*>(empty + kStages);                 // [kUsers]
    float* thr = reinterpret_cast<float*>(cnt + kUsers);                // [kUsers]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long u0 = static_cast<long long>(blockIdx.x) * kUsers;
    const int split = blockIdx.y;
    const int t0 = static_cast<int>(static_cast<long long>(p.tiles) * split / p.splits);
    const int t1 = static_cast<int>(static_cast<long long>(p.tiles) * (split + 1) / p.splits);

    if (warp == 4 && lane == 0) {
        tma_prefetch_desc(&tmUh);
        tma_prefetch_desc(&tmUl);
        tma_prefetch_desc(&tmNh);
        tma_prefetch_desc(&tmNl);
        for (int i = 0; i < kStages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 4);  // one arrival per consumer warp
        }
        fence_barrier_init();
    }
    if (threadIdx.x < kUsers) {
        cnt[threadIdx.x] = 0;
        thr[threadIdx.x] = -INFINITY;
    }
    __syncthreads();

    if (warp == 4) {
        // ===================== TMA producer: users and news boxes of every (tile, k-chunk) =====================
        if (elect_one()) {
            int st = 0;
            uint32_t ph = 0;
            for (int t = t0; t < t1; ++t)
                for (int c = 0; c < p.k_chunks; ++c) {
                    f_wait(&empty[st], ph ^ 1u, 701);
                    uint8_t* dst = sStage + st * kStage;
                    mbar_arrive_expect_tx(&full[st], kStage);  // boxes past the last row / column land zero filled
                    tma_load_2d(dst, &tmUh, &full[st], c * 64, static_cast<int>(u0));
                    tma_load_2d(dst + kBox, &tmUl, &full[st], c * 64, static_cast<int>(u0));
                    tma_load_2d(dst + 2 * kBox, &tmNh, &full[st], c * 64, t * kNews);
                    tma_load_2d(dst + 3 * kBox, &tmNl, &full[st], c * 64, t * kNews);
                    if (++st == kStages) { st = 0; ph ^= 1u; }
                }
        }
        return;
    }

    // ===================== consumer warpgroup =====================
    // exclusion rows of this tile's users are one contiguous CSR range: split 0 checks them once
    if (p.excl_offsets != nullptr && split == 0) {
        const long long uend = min(u0 + kUsers, p.n_users);
        bool bad = false;
        for (long long i = p.excl_offsets[u0] + threadIdx.x; i < p.excl_offsets[uend]; i += 128) {
            const long long r = p.excl_rows[i];
            bad |= r < 0 || r >= p.n_news;
        }
        if (bad) atomicOr(p.bad_row_flag, 1);
    }
    // fragment of m64n64: acc[4j + 2e + i] = user row 16 * warp + lane / 4 + 8e, news column 8j + 2 * (lane % 4) + i
    int urow[2];
    long long ex0[2], ex1[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        urow[e] = 16 * warp + (lane >> 2) + 8 * e;
        const long long ug = u0 + urow[e];
        ex0[e] = ex1[e] = 0;
        if (p.excl_offsets != nullptr && ug < p.n_users) {
            ex0[e] = p.excl_offsets[ug];
            ex1[e] = p.excl_offsets[ug + 1];
        }
    }
    const bool user_ok[2] = {u0 + urow[0] < p.n_users, u0 + urow[1] < p.n_users};
    const uint32_t s_base = smem_u32(sStage);
    bool bad_score = false;
    int st = 0;
    uint32_t ph = 0;
    for (int t = t0; t < t1; ++t) {
        float acc[kNews / 2];
#pragma unroll
        for (int i = 0; i < kNews / 2; ++i) acc[i] = 0.f;
        for (int c = 0; c < p.k_chunks; ++c) {
            f_wait(&full[st], ph, 702);
            const uint32_t a = s_base + st * kStage;
            const uint64_t dUh = make_sw128_desc(a, 16, 1024), dUl = make_sw128_desc(a + kBox, 16, 1024);
            const uint64_t dNh = make_sw128_desc(a + 2 * kBox, 16, 1024), dNl = make_sw128_desc(a + 3 * kBox, 16, 1024);
#pragma unroll
            for (int i = 0; i < kNews / 2; ++i) wgmma_reg_fence(acc[i]);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                Wgmma<kNews, 0, 0>::mma(acc, dUh + 2 * k, dNl + 2 * k, 1);
                Wgmma<kNews, 0, 0>::mma(acc, dUl + 2 * k, dNh + 2 * k, 1);
                Wgmma<kNews, 0, 0>::mma(acc, dUh + 2 * k, dNh + 2 * k, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < kNews / 2; ++i) wgmma_reg_fence(acc[i]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
            if (++st == kStages) { st = 0; ph ^= 1u; }
        }
        // ---- epilogue: survivors of the tile into the candidate buffers ----
        const int nrow0 = t * kNews;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            if (!user_ok[e]) continue;
            const float th = thr[urow[e]];
#pragma unroll
            for (int j = 0; j < kNews / 8; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int n = nrow0 + 8 * j + 2 * (lane & 3) + i;
                    const float s = acc[4 * j + 2 * e + i];
                    if (n >= p.n_news) continue;
                    bad_score |= !(fabsf(s) <= 3.402823466e38f);
                    if (!(s > th)) continue;
                    bool excluded = false;
                    for (long long x = ex0[e]; x < ex1[e] && !excluded; ++x) excluded = __ldg(p.excl_rows + x) == n;
                    if (excluded) continue;
                    const int pos = atomicAdd(&cnt[urow[e]], 1);
                    bs[urow[e] * kCap + pos] = s;
                    br[urow[e] * kCap + pos] = n;
                }
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
        // a buffer that could not take another tile's 64 survivors is merged down to k
        for (int u = warp; u < kUsers; u += 4)
            if (cnt[u] > kCap - kNews) merge_user(bs, br, cnt, thr, u, p.k);
        asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    if (bad_score) atomicOr(p.bad_score_flag, 1);
    // ---- the k best of every user of the tile: sorted, padded with (-inf, -1) ----
    for (int u = warp; u < kUsers; u += 4) {
        const long long ug = u0 + u;
        if (ug >= p.n_users) break;
        merge_user(bs, br, cnt, thr, u, p.k);
        const float* s = bs + u * kCap;
        const int* r = br + u * kCap;
        const int c = cnt[u];
        for (int j = lane; j < p.k; j += 32) {
            const float sv = j < c ? s[j] : -INFINITY;
            const int rv = j < c ? r[j] : -1;
            if (p.splits == 1) {
                p.idx[ug * p.k + j] = rv;
                p.score[ug * p.k + j] = sv;
            } else {
                const long long o = (ug * p.splits + split) * p.k + j;
                p.part_score[o] = sv;
                p.part_row[o] = rv;
            }
        }
    }
}

// the splits' lists of a user (one warp per user) -> its k best
constexpr int kMergeWarps = 4;
__global__ void __launch_bounds__(kMergeWarps * 32) topk_merge_kernel(const Params p) {
    __shared__ float ss[kMergeWarps][kMaxSplits * 128];
    __shared__ int sr[kMergeWarps][kMaxSplits * 128];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long u = static_cast<long long>(blockIdx.x) * kMergeWarps + w;
    if (u >= p.n_users) return;
    const int m = p.splits * p.k;
    int n = 1;
    while (n < m) n <<= 1;
    float* s = ss[w];
    int* r = sr[w];
    for (int i = lane; i < n; i += 32) {
        const float sv = i < m ? p.part_score[u * m + i] : -INFINITY;
        const int rv = i < m ? p.part_row[u * m + i] : -1;
        s[i] = sv;
        r[i] = sv == -INFINITY ? 0x7fffffff : rv;
    }
    __syncwarp();
    warp_sort(s, r, n);
    for (int j = lane; j < p.k; j += 32) {
        const bool live = s[j] != -INFINITY;
        p.idx[u * p.k + j] = live ? r[j] : -1;
        p.score[u * p.k + j] = s[j];
    }
}

}  // namespace topk

static int topk_splits(long long n_users, long long n_news) {
    const long long user_tiles = (n_users + topk::kUsers - 1) / topk::kUsers, tiles = (n_news + topk::kNews - 1) / topk::kNews;
    const long long sms = std::max(1, num_sms());
    long long s = user_tiles >= sms ? 1 : (sms + user_tiles - 1) / std::max(1ll, user_tiles);
    s = std::min<long long>({s, topk::kMaxSplits, std::max(1ll, tiles / 4)});
    return static_cast<int>(s);
}

static int topk_ld(int D) { return round_up(D, 8); }

struct TopkWorkspace : WorkspaceLayout {
    __nv_bfloat16 *uh, *ul, *nh, *nl;
    float* part_score;
    int* part_row;
    TopkWorkspace(void* base, long long n_users, long long n_news, int D, int k, int splits)
        : WorkspaceLayout{static_cast<char*>(base)} {
        const long long ld = topk_ld(D);
        uh = take<__nv_bfloat16>(n_users * ld);
        ul = take<__nv_bfloat16>(n_users * ld);
        nh = take<__nv_bfloat16>(n_news * ld);
        nl = take<__nv_bfloat16>(n_news * ld);
        part_score = take<float>(splits > 1 ? n_users * splits * k : 0);
        part_row = take<int>(splits > 1 ? n_users * splits * k : 0);
    }
};

static int topk_check(long long n_users, long long n_news, int D, int k) {
    NR_REQUIRE(k >= 1 && k <= 128, "nr_topk_dot: k=%d outside [1, 128]", k);
    NR_REQUIRE(D >= 1 && D <= 4096, "nr_topk_dot: D=%d outside [1, 4096]", D);
    NR_REQUIRE(n_users >= 0 && n_users < (1ll << 31) - topk::kUsers, "nr_topk_dot: n_users=%lld outside [0, 2^31 - 64)", n_users);
    NR_REQUIRE(n_news >= 0 && n_news < (1ll << 31) - topk::kNews, "nr_topk_dot: n_news=%lld outside [0, 2^31 - 64)", n_news);
    return 0;
}

long long topk_dot_workspace(long long n_users, long long n_news, int D, int k) {
    if (topk_check(n_users, n_news, D, k) != 0) return -1;
    return TopkWorkspace(nullptr, n_users, n_news, D, k, topk_splits(n_users, n_news)).bytes();
}

int topk_dot(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D, int k,
             const long long* excl_offsets, const long long* excl_rows, long long* idx, float* score, int* bad_row_flag,
             int* bad_score_flag, void* workspace, long long workspace_bytes, cudaStream_t stream) {
    using namespace topk;
    NR_PROPAGATE(topk_check(n_users, n_news, D, k));
    NR_REQUIRE(ld_users >= D && ld_news >= D, "nr_topk_dot: pitches ld_users=%d ld_news=%d below D=%d", ld_users, ld_news, D);
    NR_REQUIRE((excl_offsets == nullptr) == (excl_rows == nullptr), "nr_topk_dot: excl_offsets and excl_rows go together");
    const int splits = topk_splits(n_users, n_news);
    TopkWorkspace ws(workspace, n_users, n_news, D, k, splits);
    NR_REQUIRE(workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && workspace_bytes >= ws.bytes(),
               "nr_topk_dot: workspace of %lld bytes (256-byte aligned) needs %lld", workspace_bytes, ws.bytes());
    if (n_users == 0 || n_news == 0) return 0;
    const int ld = topk_ld(D);
    CUtensorMap tmUh, tmUl, tmNh, tmNl;
    NR_PROPAGATE(make_tmap_bf16_2d(&tmUh, ws.uh, n_users, D, ld, 64, kUsers));
    NR_PROPAGATE(make_tmap_bf16_2d(&tmUl, ws.ul, n_users, D, ld, 64, kUsers));
    NR_PROPAGATE(make_tmap_bf16_2d(&tmNh, ws.nh, n_news, D, ld, 64, kNews));
    NR_PROPAGATE(make_tmap_bf16_2d(&tmNl, ws.nl, n_news, D, ld, 64, kNews));
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(topk_dot_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmem)));
        attr_set = true;
    }
    const Bf16Rows jobs[2] = {
        {.src = users, .n_rows = n_users, .D = D, .s_seq = ld_users, .width = ld, .hi = ws.uh, .ld_hi = ld, .lo = ws.ul, .ld_lo = ld},
        {.src = news, .n_rows = n_news, .D = D, .s_seq = ld_news, .width = ld, .hi = ws.nh, .ld_hi = ld, .lo = ws.nl, .ld_lo = ld}};
    NR_PROPAGATE(rows_to_bf16(jobs, 2, kRowsToBf16Planes, stream));
    Params p;
    p.n_users = n_users;
    p.n_news = static_cast<int>(n_news);
    p.k = k;
    p.k_chunks = ceil_div(D, 64);
    p.tiles = static_cast<int>((n_news + kNews - 1) / kNews);
    p.splits = splits;
    p.excl_offsets = excl_offsets;
    p.excl_rows = excl_rows;
    p.idx = idx;
    p.score = score;
    p.part_score = ws.part_score;
    p.part_row = ws.part_row;
    p.bad_row_flag = bad_row_flag;
    p.bad_score_flag = bad_score_flag;
    const long long user_tiles = (n_users + kUsers - 1) / kUsers;
    {
        ProfScope ps("topk_dot", static_cast<int>(n_users), static_cast<int>(n_news), k, stream);
        topk_dot_kernel<<<dim3(static_cast<unsigned>(user_tiles), splits), kThreads, kSmem, stream>>>(tmUh, tmUl, tmNh, tmNl, p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    if (splits > 1) {
        ProfScope ps("topk_merge", static_cast<int>(n_users), splits, k, stream);
        topk_merge_kernel<<<static_cast<unsigned>((n_users + kMergeWarps - 1) / kMergeWarps), kMergeWarps * 32, 0, stream>>>(p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

}  // namespace nr
