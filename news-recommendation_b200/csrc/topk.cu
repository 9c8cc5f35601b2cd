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
//
// Ranks over the pool (nr_pool_ranks): the same planes and the same tile pipeline (DotPlanes, produce_tile, consume_tile), so
// every score is the bit pattern nr_topk_dot computes for that pair.  The CTA first runs the tiles that hold its rows'
// targets and reads the target scores out of the fragments; those are the thresholds.  In the main pass a score that does not
// come before its row's last target (the common case) is dropped; one that does, and is not a target or an exclusion of the
// row, is counted against the first target it beats (a per-row histogram; a rank is the prefix sum over the row's targets in
// output order).  Membership goes through a per-row bit filter of the targets and exclusions: a filter hit is queued and
// checked after the tile by the whole warpgroup, one entry per thread, so one lane's scan never stalls its warp.  Splits add
// integer counts, so the ranks do not depend on the order of anything.
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

// ---- the score tile pipeline of both kernels ----
// The stage ring: full[s] completes when the four boxes of stage s have landed, empty[s] when the 4 consumer warps are done.
struct Ring {
    uint8_t* stage;
    uint64_t* full;
    uint64_t* empty;
    int st = 0;
    uint32_t ph = 0;
    __device__ __forceinline__ void advance() {
        if (++st == kStages) { st = 0; ph ^= 1u; }
    }
};

// producer warp, one elected lane: prefetch the maps and initialise the ring (before the block's first __syncthreads)
__device__ __forceinline__ void ring_init(const Ring& r, const CUtensorMap* uh, const CUtensorMap* ul, const CUtensorMap* nh,
                                          const CUtensorMap* nl) {
    tma_prefetch_desc(uh);
    tma_prefetch_desc(ul);
    tma_prefetch_desc(nh);
    tma_prefetch_desc(nl);
    for (int i = 0; i < kStages; ++i) {
        mbar_init(&r.full[i], 1);
        mbar_init(&r.empty[i], 4);  // one arrival per consumer warp
    }
    fence_barrier_init();
}

// producer: the users' and news tile t's hi/lo boxes of every 64-column k-chunk, users rows [u0, u0 + 64)
__device__ __forceinline__ void produce_tile(Ring& r, const CUtensorMap* uh, const CUtensorMap* ul, const CUtensorMap* nh,
                                             const CUtensorMap* nl, int u0, int t, int k_chunks) {
    for (int c = 0; c < k_chunks; ++c) {
        f_wait(&r.empty[r.st], r.ph ^ 1u, 701);
        uint8_t* dst = r.stage + r.st * kStage;
        mbar_arrive_expect_tx(&r.full[r.st], kStage);  // boxes past the last row / column land zero filled
        tma_load_2d(dst, uh, &r.full[r.st], c * 64, u0);
        tma_load_2d(dst + kBox, ul, &r.full[r.st], c * 64, u0);
        tma_load_2d(dst + 2 * kBox, nh, &r.full[r.st], c * 64, t * kNews);
        tma_load_2d(dst + 3 * kBox, nl, &r.full[r.st], c * 64, t * kNews);
        r.advance();
    }
}

// consumer warpgroup: the 64 x 64 score tile the producer streams next, hi.lo + lo.hi + hi.hi per k16 step into acc.
// Fragment of m64n64: acc[4j + 2e + i] = user row 16 * warp + lane / 4 + 8e, news column 8j + 2 * (lane % 4) + i
__device__ __forceinline__ void consume_tile(Ring& r, float (&acc)[kNews / 2], int k_chunks) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < kNews / 2; ++i) acc[i] = 0.f;
    const uint32_t s_base = smem_u32(r.stage);
    for (int c = 0; c < k_chunks; ++c) {
        f_wait(&r.full[r.st], r.ph, 702);
        const uint32_t a = s_base + r.st * kStage;
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
        if (lane == 0) mbar_arrive(&r.empty[r.st]);
        r.advance();
    }
}

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

    Ring ring{sStage, full, empty};
    if (warp == 4 && lane == 0) ring_init(ring, &tmUh, &tmUl, &tmNh, &tmNl);
    if (threadIdx.x < kUsers) {
        cnt[threadIdx.x] = 0;
        thr[threadIdx.x] = -INFINITY;
    }
    __syncthreads();

    if (warp == 4) {
        // ===================== TMA producer: users and news boxes of every (tile, k-chunk) =====================
        if (elect_one())
            for (int t = t0; t < t1; ++t) produce_tile(ring, &tmUh, &tmUl, &tmNh, &tmNl, static_cast<int>(u0), t, p.k_chunks);
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
    // fragment rows of this thread (consume_tile)
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
    bool bad_score = false;
    for (int t = t0; t < t1; ++t) {
        float acc[kNews / 2];
        consume_tile(ring, acc, p.k_chunks);
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


// ---- ranks over the pool ----
constexpr int kMaxTargets = 32;             // targets per query row
constexpr int kFiltWords = 64;              // per row: bit (n mod 4096) set for each target and exclusion n
constexpr int kQueue = kUsers * kNews;      // a tile's filter hits, checked by the whole warpgroup after the tile
constexpr size_t kRankSmem = 1024 + kStages * kStage + kUsers * kFiltWords * 8 + 5 * kUsers * kMaxTargets * 4 + kQueue * 12 + 1024;
static_assert(kRankSmem <= 232448, "pool_ranks_kernel: shared memory");

struct RankParams {
    long long n_rows;
    int n_news, k_chunks, tiles, splits;
    const long long* tgt_offsets;   // [n_rows + 1]
    const long long* tgt_rows;
    const long long* excl_offsets;  // [n_rows + 1] or null
    const long long* excl_rows;
    long long* rank;                // [n_targets]
    float* score;
    int* part;                      // splits > 1: [n_rows][splits][kMaxTargets] counts by target slot; slot 0 = -1: bad row
    int* bad_row_flag;
    int* bad_score_flag;
    int* target_flag;
};

__global__ void __launch_bounds__(kThreads, 1) pool_ranks_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
                                                                 const __grid_constant__ CUtensorMap tmNh, const __grid_constant__ CUtensorMap tmNl,
                                                                 const RankParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sStage = base;
    unsigned long long* filt = reinterpret_cast<unsigned long long*>(sStage + kStages * kStage);  // [kUsers][kFiltWords]
    float* ts = reinterpret_cast<float*>(filt + kUsers * kFiltWords);   // [kUsers][kMaxTargets] target scores, then sorted
    int* tr = reinterpret_cast<int*>(ts + kUsers * kMaxTargets);        // target rows
    int* tp = tr + kUsers * kMaxTargets;                                // target slot in the row's CSR range
    int* hist = tp + kUsers * kMaxTargets;                              // counts by first target beaten (the sort's keys first)
    int* tiles = hist + kUsers * kMaxTargets;                           // [kUsers * kMaxTargets] pool tiles holding targets
    float* qs = reinterpret_cast<float*>(tiles + kUsers * kMaxTargets); // [kQueue] filter hits: score, news row, query row
    int* qn = reinterpret_cast<int*>(qs + kQueue);
    int* qr = qn + kQueue;
    uint64_t* full = reinterpret_cast<uint64_t*>(qr + kQueue);
    uint64_t* empty = full + kStages;
    int* tm = reinterpret_cast<int*>(empty + kStages);                  // [kUsers] targets of the row, -1: bad row
    int* n_pro = tm + kUsers;
    int* qc = n_pro + 1;                                                // [2] queue length, by tile parity
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long q0 = static_cast<long long>(blockIdx.x) * kUsers;
    const int split = blockIdx.y;
    const int t0 = static_cast<int>(static_cast<long long>(p.tiles) * split / p.splits);
    const int t1 = static_cast<int>(static_cast<long long>(p.tiles) * (split + 1) / p.splits);

    Ring ring{sStage, full, empty};
    if (warp == 4 && lane == 0) ring_init(ring, &tmQh, &tmQl, &tmNh, &tmNl);
    for (int i = threadIdx.x; i < kUsers * kFiltWords; i += kThreads) filt[i] = 0;
    if (threadIdx.x < 2) qc[threadIdx.x] = 0;
    __syncthreads();
    // ---- the rows' targets and the membership filter of targets and exclusions ----
    if (threadIdx.x < kUsers) {
        const int r = threadIdx.x;
        const long long q = q0 + r;
        int m = 0;
        if (q < p.n_rows) {
            const long long a = p.tgt_offsets[q], cnt = p.tgt_offsets[q + 1] - a;
            if (cnt > kMaxTargets) {
                m = -1;
                atomicOr(p.target_flag, 1);
            } else {
                m = static_cast<int>(cnt);
                for (int j = 0; j < m; ++j) {
                    const long long n = p.tgt_rows[a + j];
                    if (n < 0 || n >= p.n_news) {
                        m = -1;
                        break;
                    }
                    tr[r * kMaxTargets + j] = static_cast<int>(n);
                    tp[r * kMaxTargets + j] = j;
                    atomicOr(&filt[r * kFiltWords + ((n >> 6) & (kFiltWords - 1))], 1ull << (n & 63));
                }
                if (m < 0) atomicOr(p.bad_row_flag, 1);
            }
        }
        tm[r] = m;
    }
    if (p.excl_offsets != nullptr) {
        bool bad = false;
        for (int r = 0; r < kUsers && q0 + r < p.n_rows; ++r)
            for (long long i = p.excl_offsets[q0 + r] + threadIdx.x; i < p.excl_offsets[q0 + r + 1]; i += kThreads) {
                const long long n = p.excl_rows[i];
                if (n < 0 || n >= p.n_news) bad = true;
                else atomicOr(&filt[r * kFiltWords + ((n >> 6) & (kFiltWords - 1))], 1ull << (n & 63));
            }
        if (bad) atomicOr(p.bad_row_flag, 1);
    }
    __syncthreads();
    // ---- the distinct tiles holding the CTA's targets, ascending (one warp) ----
    if (warp == 0) {
        int c = 0;
        if (lane == 0)
            for (int r = 0; r < kUsers; ++r)
                for (int j = 0; j < tm[r]; ++j) tiles[c++] = tr[r * kMaxTargets + j] / kNews;
        c = __shfl_sync(0xffffffffu, c, 0);
        int n = 1;
        while (n < c) n <<= 1;
        float* keys = reinterpret_cast<float*>(hist);  // equal keys: warp_sort orders by the int
        for (int i = lane; i < n; i += 32) {
            keys[i] = 0.f;
            if (i >= c) tiles[i] = 0x7fffffff;
        }
        __syncwarp();
        warp_sort(keys, tiles, n);
        if (lane == 0) {
            int d = 0;
            for (int i = 0; i < c; ++i)
                if (d == 0 || tiles[i] != tiles[d - 1]) tiles[d++] = tiles[i];
            *n_pro = d;
        }
    }
    __syncthreads();
    const int npro = *n_pro;

    if (warp == 4) {
        // ===================== TMA producer: the target tiles, then the split's tiles =====================
        if (elect_one()) {
            for (int i = 0; i < npro; ++i) produce_tile(ring, &tmQh, &tmQl, &tmNh, &tmNl, static_cast<int>(q0), tiles[i], p.k_chunks);
            for (int t = t0; t < t1; ++t) produce_tile(ring, &tmQh, &tmQl, &tmNh, &tmNl, static_cast<int>(q0), t, p.k_chunks);
        }
        return;
    }

    // ===================== consumer warpgroup =====================
    int urow[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) urow[e] = 16 * warp + (lane >> 2) + 8 * e;
    float acc[kNews / 2];
    // prologue: the target scores, read from the fragments of the tiles that hold them
    for (int i = 0; i < npro; ++i) {
        const int t = tiles[i];
        consume_tile(ring, acc, p.k_chunks);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int r = urow[e];
            for (int j = 0; j < tm[r]; ++j) {
                const int n = tr[r * kMaxTargets + j], col = n - t * kNews;
                if (col < 0 || col >= kNews || ((col >> 1) & 3) != (lane & 3)) continue;
                float v = 0.f;
#pragma unroll
                for (int jj = 0; jj < kNews / 8; ++jj)
#pragma unroll
                    for (int ii = 0; ii < 2; ++ii)
                        if (col == 8 * jj + 2 * (lane & 3) + ii) v = acc[4 * jj + 2 * e + ii];
                ts[r * kMaxTargets + j] = v;
            }
        }
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // each row's targets into output order (score descending, row ascending); counts start at zero
    bool bad_score = false;
    if (threadIdx.x < kUsers) {
        const int r = threadIdx.x, m = tm[r];
        float* s = ts + r * kMaxTargets;
        int* n = tr + r * kMaxTargets;
        int* o = tp + r * kMaxTargets;
        for (int j = 0; j < m; ++j) bad_score |= !(fabsf(s[j]) <= 3.402823466e38f);
        for (int j = 1; j < m; ++j) {
            const float sj = s[j];
            const int nj = n[j], oj = o[j];
            int i = j;
            for (; i > 0 && before(sj, nj, s[i - 1], n[i - 1]); --i) {
                s[i] = s[i - 1];
                n[i] = n[i - 1];
                o[i] = o[i - 1];
            }
            s[i] = sj;
            n[i] = nj;
            o[i] = oj;
        }
        for (int j = 0; j < kMaxTargets; ++j) hist[r * kMaxTargets + j] = 0;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // thresholds: a score counts when it comes before the row's last target; before its first, it beats all of them
    float hi_s[2], lo_s[2];
    int hi_r[2], lo_r[2], cnt0[2] = {0, 0};
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int r = urow[e], m = tm[r];
        hi_s[e] = lo_s[e] = INFINITY;  // nothing comes before (+inf, -1)
        hi_r[e] = lo_r[e] = -1;
        if (m > 0) {
            hi_s[e] = ts[r * kMaxTargets];
            hi_r[e] = tr[r * kMaxTargets];
            lo_s[e] = ts[r * kMaxTargets + m - 1];
            lo_r[e] = tr[r * kMaxTargets + m - 1];
        }
    }
    for (int t = t0; t < t1; ++t) {
        consume_tile(ring, acc, p.k_chunks);
        const int nrow0 = t * kNews;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            if (lo_r[e] < 0) continue;  // no target, or a bad row
            const int r = urow[e];
            const unsigned long long fw = filt[r * kFiltWords + (t & (kFiltWords - 1))];
#pragma unroll
            for (int j = 0; j < kNews / 8; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int col = 8 * j + 2 * (lane & 3) + i, n = nrow0 + col;
                    const float s = acc[4 * j + 2 * e + i];
                    if (n >= p.n_news) continue;
                    bad_score |= !(fabsf(s) <= 3.402823466e38f);
                    if (!before(s, n, lo_s[e], lo_r[e])) continue;
                    if ((fw >> col) & 1ull) {  // maybe a target or an exclusion of the row: queued
                        const int k = atomicAdd(&qc[t & 1], 1);
                        qs[k] = s;
                        qn[k] = n;
                        qr[k] = r;
                        continue;
                    }
                    if (before(s, n, hi_s[e], hi_r[e])) {
                        ++cnt0[e];
                    } else {
                        int b = 1;  // the first target it comes before: exists, the last one
                        while (!before(s, n, ts[r * kMaxTargets + b], tr[r * kMaxTargets + b])) ++b;
                        atomicAdd(&hist[r * kMaxTargets + b], 1);
                    }
                }
        }
        // the queued scores, one per thread: counted unless a target or an exclusion of their row
        asm volatile("bar.sync 1, 128;" ::: "memory");
        const int nq = qc[t & 1];
        if (threadIdx.x == 0) qc[(t + 1) & 1] = 0;  // every thread read it before the previous tile's second barrier
        for (int k = threadIdx.x; k < nq; k += 128) {
            const float s = qs[k];
            const int n = qn[k], r = qr[k];
            bool member = false;
            for (int x = 0; x < tm[r] && !member; ++x) member = tr[r * kMaxTargets + x] == n;
            if (p.excl_offsets != nullptr)
                for (long long x = p.excl_offsets[q0 + r]; x < p.excl_offsets[q0 + r + 1] && !member; ++x)
                    member = __ldg(p.excl_rows + x) == n;
            if (member) continue;
            int b = 0;
            while (!before(s, n, ts[r * kMaxTargets + b], tr[r * kMaxTargets + b])) ++b;
            atomicAdd(&hist[r * kMaxTargets + b], 1);
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    if (bad_score) atomicOr(p.bad_score_flag, 1);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        int c = cnt0[e];
        c += __shfl_xor_sync(0xffffffffu, c, 1);
        c += __shfl_xor_sync(0xffffffffu, c, 2);
        if ((lane & 3) == 0 && c != 0) atomicAdd(&hist[urow[e] * kMaxTargets], c);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // ---- rank of the b-th target in output order: the counts of bins 0 .. b ----
    if (threadIdx.x < kUsers) {
        const int r = threadIdx.x, m = tm[r];
        const long long q = q0 + r;
        if (q >= p.n_rows) return;
        const long long a = p.tgt_offsets[q];
        if (m < 0) {
            if (split == 0)
                for (long long j = a; j < p.tgt_offsets[q + 1]; ++j) {
                    if (p.splits == 1) p.rank[j] = -1;
                    p.score[j] = NAN;
                }
            if (p.splits > 1) p.part[(q * p.splits + split) * kMaxTargets] = -1;
            return;
        }
        int c = 0;
        for (int b = 0; b < m; ++b) {
            c += hist[r * kMaxTargets + b];
            const int j = tp[r * kMaxTargets + b];
            if (split == 0) p.score[a + j] = ts[r * kMaxTargets + b];
            if (p.splits == 1) p.rank[a + j] = c;
            else p.part[(q * p.splits + split) * kMaxTargets + j] = c;
        }
    }
}

// the splits' counts of a row's targets (one thread per row) -> its ranks
__global__ void __launch_bounds__(128) pool_ranks_merge_kernel(const RankParams p) {
    const long long q = static_cast<long long>(blockIdx.x) * 128 + threadIdx.x;
    if (q >= p.n_rows) return;
    const long long a = p.tgt_offsets[q], cnt = p.tgt_offsets[q + 1] - a;
    const int* part = p.part + q * p.splits * kMaxTargets;
    const bool bad = cnt > kMaxTargets || (cnt > 0 && part[0] < 0);
    for (long long j = 0; j < cnt; ++j) {
        long long c = 0;
        for (int s = 0; !bad && s < p.splits; ++s) c += part[s * kMaxTargets + j];
        p.rank[a + j] = bad ? -1 : c;
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

// hi/lo bf16 planes of the users (query rows) and the news, pitch round_up(D, 8): the operands of the tile pipeline
struct DotPlanes {
    __nv_bfloat16 *uh, *ul, *nh, *nl;
    DotPlanes(WorkspaceLayout& ws, long long n_users, long long n_news, int D) {
        const long long ld = topk_ld(D);
        uh = ws.take<__nv_bfloat16>(n_users * ld);
        ul = ws.take<__nv_bfloat16>(n_users * ld);
        nh = ws.take<__nv_bfloat16>(n_news * ld);
        nl = ws.take<__nv_bfloat16>(n_news * ld);
    }
    // the four TMA maps (users hi, lo, news hi, lo), then one rows_to_bf16 launch that writes the planes
    int prepare(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D,
                CUtensorMap (&tm)[4], cudaStream_t stream) const {
        const int ld = topk_ld(D);
        NR_PROPAGATE(make_tmap_bf16_2d(&tm[0], uh, n_users, D, ld, 64, topk::kUsers));
        NR_PROPAGATE(make_tmap_bf16_2d(&tm[1], ul, n_users, D, ld, 64, topk::kUsers));
        NR_PROPAGATE(make_tmap_bf16_2d(&tm[2], nh, n_news, D, ld, 64, topk::kNews));
        NR_PROPAGATE(make_tmap_bf16_2d(&tm[3], nl, n_news, D, ld, 64, topk::kNews));
        const Bf16Rows jobs[2] = {
            {.src = users, .n_rows = n_users, .D = D, .s_seq = ld_users, .width = ld, .hi = uh, .ld_hi = ld, .lo = ul, .ld_lo = ld},
            {.src = news, .n_rows = n_news, .D = D, .s_seq = ld_news, .width = ld, .hi = nh, .ld_hi = ld, .lo = nl, .ld_lo = ld}};
        return rows_to_bf16(jobs, 2, kRowsToBf16Planes, stream);
    }
};

struct TopkWorkspace : WorkspaceLayout {
    DotPlanes planes;
    float* part_score;
    int* part_row;
    TopkWorkspace(void* base, long long n_users, long long n_news, int D, int k, int splits)
        : WorkspaceLayout{static_cast<char*>(base)}, planes(*this, n_users, n_news, D) {
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
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(topk_dot_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmem)));
        attr_set = true;
    }
    CUtensorMap tm[4];
    NR_PROPAGATE(ws.planes.prepare(users, n_users, ld_users, news, n_news, ld_news, D, tm, stream));
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
        topk_dot_kernel<<<dim3(static_cast<unsigned>(user_tiles), splits), kThreads, kSmem, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
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

struct RankWorkspace : WorkspaceLayout {
    DotPlanes planes;
    int* part;
    RankWorkspace(void* base, long long n_rows, long long n_news, int D, int splits)
        : WorkspaceLayout{static_cast<char*>(base)}, planes(*this, n_rows, n_news, D) {
        part = take<int>(splits > 1 ? n_rows * splits * topk::kMaxTargets : 0);
    }
};

static int pool_ranks_check(long long n_rows, long long n_news, int D) {
    NR_REQUIRE(D >= 1 && D <= 4096, "nr_pool_ranks: D=%d outside [1, 4096]", D);
    NR_REQUIRE(n_rows >= 0 && n_rows < (1ll << 31) - topk::kUsers, "nr_pool_ranks: n_rows=%lld outside [0, 2^31 - 64)", n_rows);
    NR_REQUIRE(n_news >= 1 && n_news < (1ll << 31) - topk::kNews, "nr_pool_ranks: n_news=%lld outside [1, 2^31 - 64)", n_news);
    return 0;
}

long long pool_ranks_workspace(long long n_rows, long long n_news, int D) {
    if (pool_ranks_check(n_rows, n_news, D) != 0) return -1;
    return RankWorkspace(nullptr, n_rows, n_news, D, topk_splits(n_rows, n_news)).bytes();
}

int pool_ranks(const float* queries, long long n_rows, int ld_queries, const float* news, long long n_news, int ld_news, int D,
               const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets, const long long* excl_rows,
               long long* rank, float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
               long long workspace_bytes, cudaStream_t stream) {
    using namespace topk;
    NR_PROPAGATE(pool_ranks_check(n_rows, n_news, D));
    NR_REQUIRE(ld_queries >= D && ld_news >= D, "nr_pool_ranks: pitches ld_queries=%d ld_news=%d below D=%d", ld_queries, ld_news, D);
    NR_REQUIRE((excl_offsets == nullptr) == (excl_rows == nullptr), "nr_pool_ranks: excl_offsets and excl_rows go together");
    const int splits = topk_splits(n_rows, n_news);
    RankWorkspace ws(workspace, n_rows, n_news, D, splits);
    NR_REQUIRE(workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && workspace_bytes >= ws.bytes(),
               "nr_pool_ranks: workspace of %lld bytes (256-byte aligned) needs %lld", workspace_bytes, ws.bytes());
    if (n_rows == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(pool_ranks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kRankSmem)));
        attr_set = true;
    }
    CUtensorMap tm[4];
    NR_PROPAGATE(ws.planes.prepare(queries, n_rows, ld_queries, news, n_news, ld_news, D, tm, stream));
    RankParams p;
    p.n_rows = n_rows;
    p.n_news = static_cast<int>(n_news);
    p.k_chunks = ceil_div(D, 64);
    p.tiles = static_cast<int>((n_news + kNews - 1) / kNews);
    p.splits = splits;
    p.tgt_offsets = tgt_offsets;
    p.tgt_rows = tgt_rows;
    p.excl_offsets = excl_offsets;
    p.excl_rows = excl_rows;
    p.rank = rank;
    p.score = score;
    p.part = ws.part;
    p.bad_row_flag = bad_row_flag;
    p.bad_score_flag = bad_score_flag;
    p.target_flag = target_flag;
    const long long row_tiles = (n_rows + kUsers - 1) / kUsers;
    {
        ProfScope ps("pool_ranks", static_cast<int>(n_rows), static_cast<int>(n_news), splits, stream);
        pool_ranks_kernel<<<dim3(static_cast<unsigned>(row_tiles), splits), kThreads, kRankSmem, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    if (splits > 1) {
        ProfScope ps("pool_ranks_merge", static_cast<int>(n_rows), splits, 0, stream);
        pool_ranks_merge_kernel<<<static_cast<unsigned>((n_rows + 127) / 128), 128, 0, stream>>>(p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

}  // namespace nr
