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
// Diversified lists (nr_topk_dot_capped): the same kernels with kCapped = true; only merge_user and the split merge change.
// The answer is the walk of the pool in output order that takes a news iff fewer than m taken news share its category and
// fewer than k are taken.  The sets with at most m news per category and at most k in all are the independent sets of a
// matroid (a partition matroid truncated to rank k), and the walk is its greedy: it takes x iff x is not spanned by the news
// ranked above it.  Spans only grow as the ground set grows, so a news the walk rejects over a set S is rejected over every
// superset of S.  Hence: (1) a merge sorts the buffer, walks it (capped_walk) and may drop every rejected entry for good;
// (2) once a merge has taken k news, a score that does not beat the k-th taken can never enter (the strict > stays), and
// while fewer than k are taken the threshold stays -inf; (3) the answer over the pool is contained in the union of the
// splits' capped lists, so the split merge sorts the union and walks it.  Two caps at once (category and subcategory) are an
// intersection of two partition matroids, which is not a matroid: a new entry could evict one whose slot then frees up, and
// (1)-(3) fail, so a call caps one field.  Shared memory is full (kSmem), so no per-entry category is kept: a merge reads
// categories[row] through the read-only path (the pool's keys stay in L2).
//
// Ranks over the pool (nr_pool_ranks): the same planes and the same tile pipeline (DotPlanes, produce_tile, consume_tile), so
// every score is the bit pattern nr_topk_dot computes for that pair.  The CTA first runs the tiles that hold its rows'
// targets and reads the target scores out of the fragments; those are the thresholds.  In the main pass a score that does not
// come before its row's last target (the common case) is dropped; one that does, and is not a target or an exclusion of the
// row, is counted against the first target it beats (a per-row histogram; a rank is the prefix sum over the row's targets in
// output order).  Membership goes through a per-row bit filter of the targets and exclusions: a filter hit is queued and
// checked after the tile by the whole warpgroup, one entry per thread, so one lane's scan never stalls its warp.  Splits add
// integer counts, so the ranks do not depend on the order of anything.
//
// MMR re-ranking (nr_mmr_rerank): one block per user re-ranks nr_topk_dot's shortlist (<= 128 entries).  The live rows are
// gathered and split into hi/lo planes in the swizzled layout the TMA boxes above have, their Gram runs on the same three
// products, and the greedy reads the Gram from shared memory.  The bounds and their derivation are in the header and DESIGN §3.
//
// List statistics (nr_list_stats): one block per list, the same live-row load, gather and Gram routines (load_live_rows,
// gram_hilo) and the same cosine (gram_sim), so a pair's similarity is the bits nr_mmr_rerank uses; the fp64 pair sums and
// the distinct-category counts are then a few hundred operations per list.
//
// Row ranges (the *_ranged entry points): query row q only sees news rows [row_lo[q], row_hi[q]).  Each CTA takes the union
// of the tiles its rows' ranges touch, [min lo / 64, ceil(max hi / 64)), and divides that interval among the splits instead
// of the pool (tile_interval, split_tiles); the epilogues drop a news outside its row's own range with one compare, where the
// unranged calls drop rows past n_news (their range is [0, n_news)).  Tile t still covers rows [64t, 64t + 64), so every
// pair's score is the bits of the unranged kernels.  The ranks kernels still run their targets' tiles first, wherever
// they are.  Without ranges the interval is [0, tiles): one code path.
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
    const int* cat;                 // capped instantiation: [n_news] category keys, at most cap news of one key per list
    int cap;
    const long long* row_lo;        // [n_users] or null: user u sees news rows [row_lo[u], row_hi[u]) only
    const long long* row_hi;
};

// a before b in the output order: higher score, then lower row
__device__ __forceinline__ bool before(float sa, int ra, float sb, int rb) { return sa > sb || (sa == sb && ra < rb); }

// The news rows [lo, hi) query row q may see: [0, n_news) without ranges; a range with lo < 0, hi > n_news or lo > hi sets
// the flag, is empty and returns false.
__device__ __forceinline__ bool row_range(const long long* row_lo, const long long* row_hi, long long q, int n_news,
                                          int* bad_row_flag, int& lo, int& hi) {
    lo = 0;
    hi = n_news;
    if (row_lo == nullptr) return true;
    const long long a = row_lo[q], b = row_hi[q];
    if (a < 0 || b > n_news || a > b) {
        atomicOr(bad_row_flag, 1);
        lo = hi = 0;
        return false;
    }
    lo = static_cast<int>(a);
    hi = static_cast<int>(b);
    return true;
}

// Threads 0..63 (two whole warps), one query row each: the union of the tiles that the non-empty ranges of the rows with
// `in` touch, per warp into iv[2 warp], iv[2 warp + 1].  The caller syncs before split_tiles reads them.
__device__ __forceinline__ void tile_interval(int lo, int hi, bool in, int* iv) {
    const bool live = in && lo < hi;
    const int a = __reduce_min_sync(~0u, live ? lo / kNews : 0x7fffffff);
    const int b = __reduce_max_sync(~0u, live ? (hi + kNews - 1) / kNews : 0);
    if ((threadIdx.x & 31) == 0) {
        iv[2 * (threadIdx.x >> 5)] = a;
        iv[2 * (threadIdx.x >> 5) + 1] = b;
    }
}

// The tiles [t0, t1) of split `split`: its share of the CTA's interval (tile_interval; [0, tiles) without ranges).  An empty
// interval gives every split no tile.
__device__ __forceinline__ void split_tiles(const int* iv, bool ranged, int tiles, int split, int splits, int& t0, int& t1) {
    int a = 0, b = tiles;
    if (ranged) {
        a = min(iv[0], iv[2]);
        b = max(iv[1], iv[3]);
        if (a >= b) a = b = 0;
    }
    const long long n = b - a;
    t0 = a + static_cast<int>(n * split / splits);
    t1 = a + static_cast<int>(n * (split + 1) / splits);
}

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

// The capped walk, one warp, over n (a multiple of 32) entries in output order, the live ones first (a dead entry has row
// INT_MAX): an entry is kept iff fewer than m earlier entries share its category and fewer than k entries before it are kept.
// The kept entries are compacted to the front, in order; returns their number (<= k <= 128).  While fewer than k are kept,
// a category's kept count is min(m, its earlier entries), so "fewer than m earlier entries" is "fewer than m among the kept
// entries of earlier chunks and the earlier entries of this chunk": the 32 lanes decide a chunk together, counting the chunk
// with __match_any_sync and the kept entries by __shfl_sync broadcasts of their categories (kept entry 32 q + l: lane l's
// kc[q]).  The categories are read through the read-only path (the pool's keys stay in L2).
__device__ int capped_walk(float* s, int* r, int n, int k, const int* __restrict__ cat, int m) {
    const int lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    int kc0 = 0, kc1 = 0, kc2 = 0, kc3 = 0;  // kc[q] (scalars: a register array indexed at run time would go to the stack)
    int kept = 0;
    for (int c0 = 0; c0 < n && kept < k; c0 += 32) {
        const float sv = s[c0 + lane];
        const int rv = r[c0 + lane];
        const bool live = rv != 0x7fffffff;
        const unsigned live_mask = __ballot_sync(~0u, live);
        if (live_mask == 0) break;
        const int cv = live ? __ldg(cat + rv) : 0;
        int same = __popc(__match_any_sync(~0u, cv) & live_mask & below);
        for (int j = 0; j < kept; ++j) {
            const int q = j >> 5;
            same += __shfl_sync(~0u, q == 0 ? kc0 : q == 1 ? kc1 : q == 2 ? kc2 : kc3, j & 31) == cv;
        }
        const unsigned take = __ballot_sync(~0u, live && same < m);
        const int nt = min(__popc(take), k - kept);
        const int pos = kept + __popc(take & below);
        __syncwarp();  // every lane has read its entry: the kept ones move down to [kept, kept + nt)
        if (((take >> lane) & 1u) && pos < kept + nt) {
            s[pos] = sv;
            r[pos] = rv;
        }
        // lane l receives new kept entry kept + t, t = (l - kept) mod 32: the category of the t-th taking lane
        const int t = (lane - kept) & 31;
        unsigned rest = take;
        for (int i = 0; i < t && rest != 0u; ++i) rest &= rest - 1u;
        const int v = __shfl_sync(~0u, cv, rest != 0u ? __ffs(rest) - 1 : lane);
        if (t < nt) {
            const int q = (kept + t) >> 5;
            if (q == 0) kc0 = v;
            else if (q == 1) kc1 = v;
            else if (q == 2) kc2 = v;
            else kc3 = v;
        }
        kept += nt;
    }
    __syncwarp();
    return kept;
}

// sorts user buffer u (pads [cnt, kCap) with (-inf, INT_MAX)), keeps the k best (capped: the k the capped walk keeps), sets
// the threshold
template <bool kCapped>
__device__ void merge_user(float* bs, int* br, int* cnt, float* thr, int u, int k, const int* cat, int m) {
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
    if constexpr (kCapped) {
        const int kept = capped_walk(s, r, kCap, k, cat, m);
        if (lane == 0) {
            cnt[u] = kept;
            thr[u] = kept >= k ? s[k - 1] : -INFINITY;
        }
    } else if (lane == 0) {
        cnt[u] = min(c, k);
        thr[u] = c >= k ? s[k - 1] : -INFINITY;
    }
    __syncwarp();
}

template <bool kCapped>
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
    int* iv = reinterpret_cast<int*>(thr + kUsers);                     // [4] tile_interval
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long u0 = static_cast<long long>(blockIdx.x) * kUsers;
    const int split = blockIdx.y;

    Ring ring{sStage, full, empty};
    if (warp == 4 && lane == 0) ring_init(ring, &tmUh, &tmUl, &tmNh, &tmNl);
    if (threadIdx.x < kUsers) {
        cnt[threadIdx.x] = 0;
        thr[threadIdx.x] = -INFINITY;
        if (p.row_lo != nullptr) {
            const long long ug = u0 + threadIdx.x;
            int lo = 0, hi = 0;
            if (ug < p.n_users) row_range(p.row_lo, p.row_hi, ug, p.n_news, p.bad_row_flag, lo, hi);
            tile_interval(lo, hi, ug < p.n_users, iv);
        }
    }
    __syncthreads();
    int t0, t1;
    split_tiles(iv, p.row_lo != nullptr, p.tiles, split, p.splits, t0, t1);

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
    int urow[2], nlo[2], nhi[2];  // the row's news range (row_range)
    long long ex0[2], ex1[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        urow[e] = 16 * warp + (lane >> 2) + 8 * e;
        const long long ug = u0 + urow[e];
        ex0[e] = ex1[e] = 0;
        nlo[e] = nhi[e] = 0;
        if (ug < p.n_users) row_range(p.row_lo, p.row_hi, ug, p.n_news, p.bad_row_flag, nlo[e], nhi[e]);
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
                    if (n < nlo[e] || n >= nhi[e]) continue;
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
            if (cnt[u] > kCap - kNews) merge_user<kCapped>(bs, br, cnt, thr, u, p.k, p.cat, p.cap);
        asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    if (bad_score) atomicOr(p.bad_score_flag, 1);
    // ---- the k best of every user of the tile: sorted, padded with (-inf, -1) ----
    for (int u = warp; u < kUsers; u += 4) {
        const long long ug = u0 + u;
        if (ug >= p.n_users) break;
        merge_user<kCapped>(bs, br, cnt, thr, u, p.k, p.cat, p.cap);
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

// the splits' lists of a user (one warp per user) -> its k best (capped: the union's capped walk, which contains the answer
// over the whole pool, since every split's list does over its part)
constexpr int kMergeWarps = 4;
template <bool kCapped>
__global__ void __launch_bounds__(kMergeWarps * 32) topk_merge_kernel(const Params p) {
    __shared__ float ss[kMergeWarps][kMaxSplits * 128];
    __shared__ int sr[kMergeWarps][kMaxSplits * 128];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long u = static_cast<long long>(blockIdx.x) * kMergeWarps + w;
    if (u >= p.n_users) return;
    const int m = p.splits * p.k;
    int n = kCapped ? 32 : 1;  // the capped walk takes whole 32-entry chunks
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
    if constexpr (kCapped) {
        const int kept = capped_walk(s, r, n, p.k, p.cat, p.cap);
        for (int j = lane; j < p.k; j += 32) {
            p.idx[u * p.k + j] = j < kept ? r[j] : -1;
            p.score[u * p.k + j] = j < kept ? s[j] : -INFINITY;
        }
    } else {
        for (int j = lane; j < p.k; j += 32) {
            const bool live = s[j] != -INFINITY;
            p.idx[u * p.k + j] = live ? r[j] : -1;
            p.score[u * p.k + j] = s[j];
        }
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
    const long long* row_lo;        // [n_rows] or null: row q counts news rows [row_lo[q], row_hi[q]) only
    const long long* row_hi;
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
    int* rlo = qc + 2;                                                  // [kUsers] the row's news range (row_range)
    int* rhi = rlo + kUsers;
    int* iv = rhi + kUsers;                                             // [4] tile_interval
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long q0 = static_cast<long long>(blockIdx.x) * kUsers;
    const int split = blockIdx.y;

    Ring ring{sStage, full, empty};
    if (warp == 4 && lane == 0) ring_init(ring, &tmQh, &tmQl, &tmNh, &tmNl);
    for (int i = threadIdx.x; i < kUsers * kFiltWords; i += kThreads) filt[i] = 0;
    if (threadIdx.x < 2) qc[threadIdx.x] = 0;
    __syncthreads();
    // ---- the rows' targets and the membership filter of targets and exclusions ----
    if (threadIdx.x < kUsers) {
        const int r = threadIdx.x;
        const long long q = q0 + r;
        int m = 0, lo = 0, hi = 0;
        if (q < p.n_rows) {
            const bool ok = row_range(p.row_lo, p.row_hi, q, p.n_news, p.bad_row_flag, lo, hi);
            const long long a = p.tgt_offsets[q], cnt = p.tgt_offsets[q + 1] - a;
            if (cnt > kMaxTargets) {
                m = -1;
                atomicOr(p.target_flag, 1);
            } else if (!ok) {
                m = -1;
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
        rlo[r] = lo;
        rhi[r] = hi;
        if (p.row_lo != nullptr) tile_interval(lo, hi, m > 0, iv);
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
    int t0, t1;
    split_tiles(iv, p.row_lo != nullptr, p.tiles, split, p.splits, t0, t1);

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
    int hi_r[2], lo_r[2], cnt0[2] = {0, 0}, nlo[2], nhi[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int r = urow[e], m = tm[r];
        nlo[e] = rlo[r];
        nhi[e] = rhi[r];
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
                    if (n < nlo[e] || n >= nhi[e]) continue;
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

// ---- maximal-marginal-relevance re-ranking of a shortlist (nr_mmr_rerank) ----
constexpr int kMmrDepth = 128;                 // shortlist entries per user, at most
constexpr int kMmrThreads = 256;               // two warpgroups: Gram rows [0, 64) and [64, 128)
constexpr int kMmrPlane = kMmrDepth * 128;     // one 64-column chunk of 128 rows, bf16, 128-byte swizzled (two kBox)
constexpr int kMmrGramLd = kMmrDepth + 8;      // fp32 Gram pitch: the fragment stores and the row reads are conflict free
constexpr size_t kMmrBuf = 2 * 2 * kMmrPlane;  // two chunk buffers of hi | lo planes
constexpr size_t kMmrGram = size_t(kMmrDepth) * kMmrGramLd * 4;  // aliases the buffers once the last chunk is done
constexpr size_t kMmrSmem = 1024 + (kMmrBuf > kMmrGram ? kMmrBuf : kMmrGram) + 1024;
static_assert(kMmrSmem <= 232448, "mmr_rerank_kernel: shared memory");

// the rows whose Gram one block computes: fp32 [.][ld], D columns in k_chunks blocks of 64
struct GramRows {
    const float* news;
    int ld, D, k_chunks;
    bool vec4;                // news and ld allow 16-byte loads
};

struct MmrParams {
    GramRows src;
    long long n_news, n_users;
    int depth, k;
    float lam, one_minus_lam;
    const long long* sl_idx;  // [n_users][depth] nr_topk_dot's list
    const float* sl_score;
    long long* idx;           // [n_users][k]
    float* score;
    int* bad_row_flag;
};

// the live entries of one list of len <= 128 (those before the first -1) into rows, all threads: a row outside [0, n_news)
// sets the flag and reads as zeros (-1).  Returns the number of live entries.
__device__ __forceinline__ int load_live_rows(const long long* list, int len, long long n_news, int* rows, int* s_live,
                                              int* bad_row_flag) {
    const int tid = threadIdx.x;
    if (tid == 0) *s_live = len;
    __syncthreads();
    const long long r = tid < len ? list[tid] : -1;
    if (tid < len && r == -1) atomicMin(s_live, tid);
    __syncthreads();
    const int live = *s_live;
    if (tid < live) {
        const bool ok = r >= 0 && r < n_news;
        if (!ok) atomicOr(bad_row_flag, 1);
        rows[tid] = ok ? static_cast<int>(r) : -1;
    }
    __syncthreads();
    return live;
}

// chunk c (columns [64c, 64c + 64)) of the list's rows into hi / lo planes, rows at and past live zero: thread t
// converts the 16-byte pieces t, t + 256, ... (row q / 8, piece q % 8, which lands at piece (q % 8) ^ (row % 8))
__device__ __forceinline__ void gram_gather_chunk(const GramRows& p, const int* rows, int live, int c, uint8_t* buf) {
    for (int q = threadIdx.x; q < kMmrDepth * 8; q += kMmrThreads) {
        const int r = q >> 3, j = q & 7, col0 = c * 64 + 8 * j;
        float x[8];
        const int row = r < live ? rows[r] : -1;
        const float* src = p.news + static_cast<long long>(row < 0 ? 0 : row) * p.ld + col0;
        if (row >= 0 && p.vec4 && col0 + 8 <= p.D) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src + 4));
            x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
            x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] = row >= 0 && col0 + e < p.D ? __ldg(src + e) : 0.f;
        }
        uint32_t h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float h0 = bf16_round(x[2 * e]), h1 = bf16_round(x[2 * e + 1]);
            h[e] = pack_bf16x2(h0, h1);
            l[e] = pack_bf16x2(x[2 * e] - h0, x[2 * e + 1] - h1);
        }
        const int off = r * 128 + ((j ^ (r & 7)) << 4);
        *reinterpret_cast<uint4*>(buf + off) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(buf + kMmrPlane + off) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

// all 256 threads: the Gram G[i][j] = hi_i.lo_j + lo_i.hi_j + hi_i.hi_j of the first live rows (rows past live are zeros)
// on wgmma, m64n128 per warpgroup, the gather of chunk c + 1 under the MMAs of chunk c; G [kMmrDepth][kMmrGramLd] fp32
// overwrites the chunk buffers at base and is complete for every thread on return
__device__ __forceinline__ void gram_hilo(const GramRows& p, const int* rows, int live, uint8_t* base) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    float* G = reinterpret_cast<float*>(base);
    float acc[kMmrDepth / 2];
#pragma unroll
    for (int i = 0; i < kMmrDepth / 2; ++i) acc[i] = 0.f;
    gram_gather_chunk(p, rows, live, 0, base);
    fence_proxy_async();
    __syncthreads();
    // every warpgroup issues its MMAs on every chunk (rows past live are zeros): a warpgroup-divergent wgmma is serialised
    for (int c = 0; c < p.k_chunks; ++c) {
        const uint32_t a = smem_u32(base + (c & 1) * 2 * kMmrPlane);
        const uint64_t dAh = make_sw128_desc(a + wg * kBox, 16, 1024), dAl = make_sw128_desc(a + kMmrPlane + wg * kBox, 16, 1024);
        const uint64_t dBh = make_sw128_desc(a, 16, 1024), dBl = make_sw128_desc(a + kMmrPlane, 16, 1024);
#pragma unroll
        for (int i = 0; i < kMmrDepth / 2; ++i) wgmma_reg_fence(acc[i]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            Wgmma<kMmrDepth, 0, 0>::mma(acc, dAh + 2 * k, dBl + 2 * k, 1);
            Wgmma<kMmrDepth, 0, 0>::mma(acc, dAl + 2 * k, dBh + 2 * k, 1);
            Wgmma<kMmrDepth, 0, 0>::mma(acc, dAh + 2 * k, dBh + 2 * k, 1);
        }
        wgmma_commit();
        // the other buffer was last read by chunk c - 1's MMAs, which every warpgroup waited for before the barrier
        if (c + 1 < p.k_chunks) gram_gather_chunk(p, rows, live, c + 1, base + ((c + 1) & 1) * 2 * kMmrPlane);
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < kMmrDepth / 2; ++i) wgmma_reg_fence(acc[i]);
        fence_proxy_async();
        __syncthreads();
    }
    // fragment of m64n128 (nr_wgmma.cuh): acc[4j + 2e + i] = row 64 wg + 16 (warp % 4) + lane / 4 + 8e, column 8j + 2 (lane % 4) + i
#pragma unroll
    for (int j = 0; j < kMmrDepth / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int row = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * e, col = 8 * j + 2 * (lane & 3);
            *reinterpret_cast<float2*>(G + row * kMmrGramLd + col) = make_float2(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]);
        }
    __syncthreads();
}

// 1 / |x_i| from the Gram's diagonal, 0 for a zero row
__device__ __forceinline__ float gram_rnorm(float g_ii) { return g_ii > 0.f ? __frsqrt_rn(g_ii) : 0.f; }

// sim(i, j) = (G_ji rsqrt(G_jj)) rsqrt(G_ii), each product rounded on its own (the cosine of nr_mmr_rerank and nr_list_stats)
__device__ __forceinline__ float gram_sim(float g_ji, float rn_j, float rn_i) { return __fmul_rn(__fmul_rn(g_ji, rn_j), rn_i); }

// one block per user: the Gram of the live rows (gram_hilo), then the greedy on warpgroup 0, one thread per shortlist position
__global__ void __launch_bounds__(kMmrThreads) mmr_rerank_kernel(const MmrParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const float* G = reinterpret_cast<const float*>(base);  // [kMmrDepth][kMmrGramLd], after gram_hilo
    __shared__ int rows[kMmrDepth];
    __shared__ float rn[kMmrDepth];                    // 1 / |row| from the diagonal, 0 for a zero row
    __shared__ float red_s[2][4];                      // per-warp (objective or score) and position of a step
    __shared__ int red_i[2][4];
    __shared__ int s_live;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const long long u = blockIdx.x;
    const long long* sl_idx = p.sl_idx + u * p.depth;
    const float* sl_score = p.sl_score + u * p.depth;

    const int live = load_live_rows(sl_idx, p.depth, p.n_news, rows, &s_live, p.bad_row_flag);
    gram_hilo(p.src, rows, live, base);
    if (wg != 0) return;

    // ---- relevance: (s_i - s_min) / (s_max - s_min) over the live entries, 1 when they are all equal ----
    const int i = tid;
    const bool is_live = i < live;
    const float s = is_live ? sl_score[i] : 0.f;
    float smax = is_live ? s : -INFINITY, smin = is_live ? s : INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        smax = fmaxf(smax, __shfl_xor_sync(~0u, smax, o));
        smin = fminf(smin, __shfl_xor_sync(~0u, smin, o));
    }
    if (lane == 0) {
        red_s[0][warp] = smax;
        red_s[1][warp] = smin;
    }
    if (is_live) {
        rn[i] = gram_rnorm(G[i * kMmrGramLd + i]);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    smax = fmaxf(fmaxf(red_s[0][0], red_s[0][1]), fmaxf(red_s[0][2], red_s[0][3]));
    smin = fminf(fminf(red_s[1][0], red_s[1][1]), fminf(red_s[1][2], red_s[1][3]));
    const float rel = smax == smin ? 1.f : __fdiv_rn(__fsub_rn(s, smin), __fsub_rn(smax, smin));
    const float rn_i = is_live ? rn[i] : 0.f;
    asm volatile("bar.sync 1, 128;" ::: "memory");  // red_s is reused by the steps

    // ---- greedy: obj_i = lam rel_i - (1 - lam) max_{j in S} sim(i, j) (0 over the empty S), the largest wins, equal
    // objectives go to the lower position; every product and difference is rounded on its own (no contraction), so lam = 1
    // gives obj = rel exactly ----
    const int picks = min(p.k, live);
    bool taken = !is_live;
    float msim = 0.f;
    long long* out_idx = p.idx + u * p.k;
    float* out_score = p.score + u * p.k;
    for (int t = 0; t < picks; ++t) {
        // a taken or dead entry is (-inf, i + 128): it loses to every open one, and best is always a position
        float ob = taken ? -INFINITY : __fsub_rn(__fmul_rn(p.lam, rel), __fmul_rn(p.one_minus_lam, msim));
        if (ob != ob) ob = -INFINITY;  // only a non-finite input gets here
        int pos = taken ? i + 128 : i;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob2 = __shfl_xor_sync(~0u, ob, o);
            const int pos2 = __shfl_xor_sync(~0u, pos, o);
            if (ob2 > ob || (ob2 == ob && pos2 < pos)) {
                ob = ob2;
                pos = pos2;
            }
        }
        if (lane == 0) {
            red_s[t & 1][warp] = ob;
            red_i[t & 1][warp] = pos;
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");  // one barrier per step: the slots alternate
        int best = red_i[t & 1][0];
        float bo = red_s[t & 1][0];
#pragma unroll
        for (int w = 1; w < 4; ++w) {
            const float o2 = red_s[t & 1][w];
            const int p2 = red_i[t & 1][w];
            if (o2 > bo || (o2 == bo && p2 < best)) {
                bo = o2;
                best = p2;
            }
        }
        best &= kMmrDepth - 1;
        if (i == best) {
            taken = true;
            out_idx[t] = sl_idx[i];
            out_score[t] = s;
        }
        // sim(i, best) = (G[best][i] / |best|) / |i|: row best of the Gram
        const float sim = gram_sim(G[best * kMmrGramLd + i], rn[best], rn_i);
        msim = t == 0 ? sim : fmaxf(msim, sim);
    }
    for (int t = picks + i; t < p.k; t += 128) {
        out_idx[t] = -1;
        out_score[t] = -INFINITY;
    }
}

// ---- per-list similarity and category statistics (nr_list_stats) ----
constexpr int kListMaxKs = 8;  // cut-offs per call

struct ListStatsParams {
    GramRows src;
    long long n_news;
    const long long* idx;      // [n_rows][k]
    const int* categories;     // [n_news] or null
    int k, n_ks, k_max;        // k_max = ks[n_ks - 1]
    int ks[kListMaxKs];        // ascending, in [1, k]
    double* pair_sum;          // [n_rows][n_ks]
    int* distinct;             // [n_rows][n_ks], null iff categories is
    int* bad_row_flag;
};

// one block per list: the Gram of the entries the largest cut-off reads (gram_hilo, as nr_mmr_rerank), then thread j sums
// sim(i, j) over i < j in fp64 (i ascending) and marks whether its category is new among entries 0 .. j; thread c of the
// cut-offs adds those up over j < K' (j ascending)
__global__ void __launch_bounds__(kMmrThreads) list_stats_kernel(const ListStatsParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const float* G = reinterpret_cast<const float*>(base);  // [kMmrDepth][kMmrGramLd], after gram_hilo
    __shared__ int rows[kMmrDepth];
    __shared__ float rn[kMmrDepth];
    __shared__ double row_sum[kMmrDepth];              // sum_{i < j} sim(i, j)
    __shared__ int cat[kMmrDepth];
    __shared__ int is_new[kMmrDepth];                  // entry j's category is not among entries 0 .. j - 1
    __shared__ int s_live;
    const int tid = threadIdx.x;
    const long long r = blockIdx.x;

    const int live = load_live_rows(p.idx + r * p.k, p.k, p.n_news, rows, &s_live, p.bad_row_flag);
    const int used = min(live, p.k_max);               // block-uniform
    if (used >= 2) {
        gram_hilo(p.src, rows, used, base);
        if (tid < used) rn[tid] = gram_rnorm(G[tid * kMmrGramLd + tid]);
    }
    if (p.categories && tid < used) cat[tid] = rows[tid] >= 0 ? __ldg(p.categories + rows[tid]) : 0;
    __syncthreads();
    if (tid < used) {
        const int j = tid;
        double s = 0.0;
        if (used >= 2) {
            const float rn_j = rn[j];
            for (int i = 0; i < j; ++i) s += static_cast<double>(gram_sim(G[j * kMmrGramLd + i], rn_j, rn[i]));
        }
        row_sum[j] = s;
        if (p.categories) {
            const int c = cat[j];
            int fresh = 1;
            for (int i = 0; i < j; ++i) fresh &= cat[i] != c;
            is_new[j] = fresh;
        }
    }
    __syncthreads();
    if (tid < p.n_ks) {
        int K = 0;
#pragma unroll
        for (int c = 0; c < kListMaxKs; ++c) K = c == tid ? p.ks[c] : K;  // no dynamic index into the parameters
        const int kk = min(K, live);
        double s = 0.0;
        int d = 0;
        for (int j = 0; j < kk; ++j) s += row_sum[j];
        p.pair_sum[r * p.n_ks + tid] = s;
        if (p.categories) {
            for (int j = 0; j < kk; ++j) d += is_new[j];
            p.distinct[r * p.n_ks + tid] = d;
        }
    }
}

// ---- the archive DNN scorer over the pool (nr_topk_archive, nr_pool_ranks_archive) ----
// score(u, n) = b2 + sum_j w2_j relu(X[n][j] + sum_p w_p Y[u p][j]),  w = softmax_p(A_u[p] . c_n),  X = W1c c + b1, Y = W1u A_u[p].
// A CTA owns G = 64 / P users, i.e. the G P archive rows [u0 P, u0 P + G P) as the wgmma M side of the tile pipeline above
// (produce_tile / consume_tile at row offset u0 P); the 64 x 64 logit tile goes to shared memory and the consumer warpgroup
// scores the tile's G x 64 pairs against the tile's X rows and the CTA's Y rows, both staged in shared memory.  P = 1 (DKN)
// has w = 1 and runs no TMA ring and no wgmma.
constexpr int kArchMaxP = 32;            // archive rows per user
constexpr int kArchMaxHid = 32;          // DNN hidden width
constexpr int kArchTileLd = kNews + 8;   // fp32 pitch of the logit / score tile

struct ArchOperands {
    int P, G, hid, hp;                   // archive rows per user, users per CTA, hidden width, hidden rounded up to 8
    const float* X;                      // [n_news][hp]          W1[:, :F] c + b1, zeros past hid
    const float* Y;                      // [n_users * P][hp]     W1[:, F:] a, zeros past hid
    const float* w2;                     // [hid]
    const float* b2;                     // [1]
};

// Shared memory of the archive kernels, byte offsets from the 1024-aligned base: the TMA ring (P > 1), the logit / score
// tile, the per-thread softmax weights (P > 1), the tile's X rows (pitch hp + 4: conflict-free 16-byte reads), the CTA's
// Y rows, w2 | b2, then the kernel's own region of `rest` bytes.
struct ArchSmem {
    int tile, w, x, y, w2, rest, bytes;
    __host__ __device__ constexpr ArchSmem(int P, int G, int hp, int rest_bytes) {
        tile = P > 1 ? kStages * kStage : 0;
        w = tile + kUsers * kArchTileLd * 4;
        x = w + (P > 1 ? kArchMaxP * 128 * 4 : 0);
        y = x + kNews * (hp + 4) * 4;
        w2 = y + G * P * hp * 4;
        rest = w2 + (kArchMaxHid + 4) * 4;
        bytes = rest + rest_bytes;
    }
};
__host__ __device__ constexpr int topk_archive_rest(int G) { return G * kCap * 8 + 2 * kStages * 8 + 4 * kUsers * 4 + 16; }
__host__ __device__ constexpr int ranks_archive_rest(int G) {
    // hist and tiles hold kUsers * kMaxTargets entries: the tile sort needs a power of two
    return G * kFiltWords * 8 + 3 * G * kMaxTargets * 4 + 2 * kUsers * kMaxTargets * 4 + 3 * G * kNews * 4 + 2 * kStages * 8 +
           5 * G * 4 + 32;
}

// X or Y: out[r][j] = (sum_f W[j][f] src[r][f]) (+ b[j]) for j < hid, in f order, 0 for hid <= j < hp; one warp per row
__global__ void __launch_bounds__(256) arch_project_kernel(const float* __restrict__ src, long long rows, int F,
                                                           const float* __restrict__ W, int ldw, const float* __restrict__ b,
                                                           int hid, int hp, float* __restrict__ out) {
    const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
    const int j = threadIdx.x & 31;
    if (r >= rows || j >= hp) return;
    float acc = 0.f;
    if (j < hid) {
        const float* w = W + static_cast<long long>(j) * ldw;
        const float* x = src + r * F;
        for (int f = 0; f < F; ++f) acc = __fmaf_rn(__ldg(w + f), __ldg(x + f), acc);
        if (b != nullptr) acc = __fadd_rn(acc, __ldg(b + j));
    }
    out[r * hp + j] = acc;
}

// THE score of one pair, in one fixed operation order (both kernels call it, so a pair has the same bits in both):
//   m = max_p l_p;  e_p = __expf(l_p - m);  z = ((e_0 + e_1) + ...) + e_{P-1};  w_p = e_p rcp_rn(z)        (P = 1: w_0 = 1)
//   pre_j = fma(w_{P-1}, Y_{P-1,j}, ... fma(w_0, Y_0j, X_j));  out = fma(w2_{hp-1}, relu(pre_{hp-1}), ... fma(w2_0, relu(pre_0), b2))
// lg: the pair's logit column (rows p of pitch kArchTileLd); xr: the news' X row; yr: the user's P Y rows (pitch hp); ws: the
// thread's weight slots (stride 128).  relu keeps a NaN, so a non-finite operand gives a non-finite score.
__device__ __forceinline__ float arch_pair_score(const float* lg, const float* xr, const float* yr, const float* w2, float b2,
                                                 float* ws, int P, int hp) {
    if (P > 1) {
        float m = lg[0];
        for (int p = 1; p < P; ++p) m = fmaxf(m, lg[p * kArchTileLd]);
        float z = 0.f;
        for (int p = 0; p < P; ++p) {
            const float e = __expf(__fsub_rn(lg[p * kArchTileLd], m));
            ws[p * 128] = e;
            z = __fadd_rn(z, e);
        }
        const float rz = __frcp_rn(z);
        for (int p = 0; p < P; ++p) ws[p * 128] = __fmul_rn(ws[p * 128], rz);
    }
    float out = b2;
    for (int jb = 0; jb < hp; jb += 8) {
        const float4 xa = *reinterpret_cast<const float4*>(xr + jb), xb = *reinterpret_cast<const float4*>(xr + jb + 4);
        float a[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
        for (int p = 0; p < P; ++p) {
            const float w = P > 1 ? ws[p * 128] : 1.f;
            const float4 ya = *reinterpret_cast<const float4*>(yr + p * hp + jb);
            const float4 yb = *reinterpret_cast<const float4*>(yr + p * hp + jb + 4);
            a[0] = __fmaf_rn(w, ya.x, a[0]);
            a[1] = __fmaf_rn(w, ya.y, a[1]);
            a[2] = __fmaf_rn(w, ya.z, a[2]);
            a[3] = __fmaf_rn(w, ya.w, a[3]);
            a[4] = __fmaf_rn(w, yb.x, a[4]);
            a[5] = __fmaf_rn(w, yb.y, a[5]);
            a[6] = __fmaf_rn(w, yb.z, a[6]);
            a[7] = __fmaf_rn(w, yb.w, a[7]);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) out = __fmaf_rn(w2[jb + i], a[i] < 0.f ? 0.f : a[i], out);
    }
    return out;
}

// Per tile, consumer warpgroup: (P > 1) the logits of news tile t into T; the tile's X rows into Xs.  The caller syncs.
__device__ __forceinline__ void arch_stage_tile(Ring& r, const ArchOperands& o, int t, int n_news, int k_chunks, float* T, float* Xs) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (o.P > 1) {
        float acc[kNews / 2];
        consume_tile(r, acc, k_chunks);
#pragma unroll
        for (int j = 0; j < kNews / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int row = 16 * warp + (lane >> 2) + 8 * e, col = 8 * j + 2 * (lane & 3);
                *reinterpret_cast<float2*>(T + row * kArchTileLd + col) = make_float2(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]);
            }
    }
    const int q4 = o.hp / 4;
    for (int i = threadIdx.x; i < kNews * q4; i += 128) {
        const int row = i / q4, q = i - row * q4;
        const long long n = static_cast<long long>(t) * kNews + row;
        const float4 v = n < n_news ? __ldg(reinterpret_cast<const float4*>(o.X + n * o.hp) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(Xs + row * (o.hp + 4) + 4 * q) = v;
    }
}

// Every (user g < here, column c) pair of the staged tile, scored and handed to visit(g, c, s): thread i takes column i % 64
// and users i / 64, i / 64 + 2, ... (a warp shares its user: the Y reads are broadcasts)
template <class Visit>
__device__ __forceinline__ void arch_tile_pairs(const ArchOperands& o, const float* T, const float* Xs, const float* Ys,
                                                const float* w2s, float* Ws, int here, Visit&& visit) {
    const int c = threadIdx.x & (kNews - 1);
    const float b2 = w2s[kArchMaxHid];
    for (int g = threadIdx.x >> 6; g < here; g += 2)
        visit(g, c, arch_pair_score(T + g * o.P * kArchTileLd + c, Xs + c * (o.hp + 4), Ys + g * o.P * o.hp, w2s, b2,
                                    Ws + threadIdx.x, o.P, o.hp));
}

// Y rows of users [u0, u0 + here) and w2 | b2 into shared memory (all threads; the caller syncs)
__device__ __forceinline__ void arch_stage_users(const ArchOperands& o, long long u0, int here, float* Ys, float* w2s) {
    const long long y0 = u0 * o.P * o.hp;
    for (int i = threadIdx.x; i < o.G * o.P * o.hp; i += kThreads) Ys[i] = i < here * o.P * o.hp ? __ldg(o.Y + y0 + i) : 0.f;
    for (int i = threadIdx.x; i < kArchMaxHid; i += kThreads) w2s[i] = i < o.hid ? __ldg(o.w2 + i) : 0.f;
    if (threadIdx.x == 0) w2s[kArchMaxHid] = __ldg(o.b2);
}

template <bool kCapped>
__global__ void __launch_bounds__(kThreads, 1) topk_archive_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                                                                   const __grid_constant__ CUtensorMap tmNh, const __grid_constant__ CUtensorMap tmNl,
                                                                   const Params p, const ArchOperands o) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int G = o.G;
    const ArchSmem L(o.P, G, o.hp, topk_archive_rest(G));
    float* T = reinterpret_cast<float*>(base + L.tile);
    float* Ws = reinterpret_cast<float*>(base + L.w);
    float* Xs = reinterpret_cast<float*>(base + L.x);
    float* Ys = reinterpret_cast<float*>(base + L.y);
    float* w2s = reinterpret_cast<float*>(base + L.w2);
    float* bs = reinterpret_cast<float*>(base + L.rest);            // [G][kCap] candidate scores
    int* br = reinterpret_cast<int*>(bs + G * kCap);                // [G][kCap] candidate rows
    uint64_t* full = reinterpret_cast<uint64_t*>(br + G * kCap);    // [kStages]
    uint64_t* empty = full + kStages;                               // [kStages]
    int* cnt = reinterpret_cast<int*>(empty + kStages);             // [G]
    float* thr = reinterpret_cast<float*>(cnt + kUsers);            // [G]
    int* rlo = reinterpret_cast<int*>(thr + kUsers);                // [G] the user's news range (row_range)
    int* rhi = rlo + kUsers;
    int* iv = rhi + kUsers;                                         // [4] tile_interval
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long u0 = static_cast<long long>(blockIdx.x) * G;
    const int here = static_cast<int>(min(static_cast<long long>(G), p.n_users - u0));
    const int split = blockIdx.y;

    Ring ring{base, full, empty};
    if (o.P > 1 && warp == 4 && lane == 0) ring_init(ring, &tmAh, &tmAl, &tmNh, &tmNl);
    if (threadIdx.x < kUsers) {
        const int g = threadIdx.x;
        int lo = 0, hi = 0;
        if (g < here) row_range(p.row_lo, p.row_hi, u0 + g, p.n_news, p.bad_row_flag, lo, hi);
        if (g < G) {
            cnt[g] = 0;
            thr[g] = -INFINITY;
            rlo[g] = lo;
            rhi[g] = hi;
        }
        if (p.row_lo != nullptr) tile_interval(lo, hi, g < here, iv);
    }
    arch_stage_users(o, u0, here, Ys, w2s);
    __syncthreads();
    int t0, t1;
    split_tiles(iv, p.row_lo != nullptr, p.tiles, split, p.splits, t0, t1);

    if (warp == 4) {
        // ===================== TMA producer (P > 1): archive rows [u0 P, u0 P + 64) and the news of every tile =====================
        if (o.P > 1 && elect_one())
            for (int t = t0; t < t1; ++t) produce_tile(ring, &tmAh, &tmAl, &tmNh, &tmNl, static_cast<int>(u0 * o.P), t, p.k_chunks);
        return;
    }

    // ===================== consumer warpgroup =====================
    if (p.excl_offsets != nullptr && split == 0) {
        bool bad = false;
        for (long long i = p.excl_offsets[u0] + threadIdx.x; i < p.excl_offsets[u0 + here]; i += 128) {
            const long long r = p.excl_rows[i];
            bad |= r < 0 || r >= p.n_news;
        }
        if (bad) atomicOr(p.bad_row_flag, 1);
    }
    bool bad_score = false;
    for (int t = t0; t < t1; ++t) {
        arch_stage_tile(ring, o, t, p.n_news, p.k_chunks, T, Xs);
        asm volatile("bar.sync 1, 128;" ::: "memory");
        // ---- survivors of the tile into the candidate buffers ----
        arch_tile_pairs(o, T, Xs, Ys, w2s, Ws, here, [&](int g, int c, float s) {
            const int n = t * kNews + c;
            if (n < rlo[g] || n >= rhi[g]) return;
            bad_score |= !(fabsf(s) <= 3.402823466e38f);
            if (!(s > thr[g])) return;
            if (p.excl_offsets != nullptr) {
                const long long x1 = p.excl_offsets[u0 + g + 1];
                for (long long x = p.excl_offsets[u0 + g]; x < x1; ++x)
                    if (__ldg(p.excl_rows + x) == n) return;
            }
            const int pos = atomicAdd(&cnt[g], 1);
            bs[g * kCap + pos] = s;
            br[g * kCap + pos] = n;
        });
        asm volatile("bar.sync 1, 128;" ::: "memory");
        for (int u = warp; u < here; u += 4)
            if (cnt[u] > kCap - kNews) merge_user<kCapped>(bs, br, cnt, thr, u, p.k, p.cat, p.cap);
        asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    if (bad_score) atomicOr(p.bad_score_flag, 1);
    // ---- the k best of every user of the CTA: sorted, padded with (-inf, -1) ----
    for (int u = warp; u < here; u += 4) {
        const long long ug = u0 + u;
        merge_user<kCapped>(bs, br, cnt, thr, u, p.k, p.cat, p.cap);
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
                const long long off = (ug * p.splits + split) * p.k + j;
                p.part_score[off] = sv;
                p.part_row[off] = rv;
            }
        }
    }
}

// nr_pool_ranks_kernel's algorithm over the CTA's G users, on the archive scores: the target tiles first (their scores read
// out of the score tile), then the split's tiles, each pair counted against the first target it comes before
__global__ void __launch_bounds__(kThreads, 1) pool_ranks_archive_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                                                                         const __grid_constant__ CUtensorMap tmNh, const __grid_constant__ CUtensorMap tmNl,
                                                                         const RankParams p, const ArchOperands o) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int G = o.G;
    const ArchSmem L(o.P, G, o.hp, ranks_archive_rest(G));
    float* T = reinterpret_cast<float*>(base + L.tile);
    float* Ws = reinterpret_cast<float*>(base + L.w);
    float* Xs = reinterpret_cast<float*>(base + L.x);
    float* Ys = reinterpret_cast<float*>(base + L.y);
    float* w2s = reinterpret_cast<float*>(base + L.w2);
    unsigned long long* filt = reinterpret_cast<unsigned long long*>(base + L.rest);  // [G][kFiltWords]
    float* ts = reinterpret_cast<float*>(filt + G * kFiltWords);    // [G][kMaxTargets] target scores, then sorted
    int* tr = reinterpret_cast<int*>(ts + G * kMaxTargets);         // target rows
    int* tp = tr + G * kMaxTargets;                                 // target slot in the row's CSR range
    int* hist = tp + G * kMaxTargets;                               // counts by first target beaten (the sort's keys first)
    int* tiles = hist + kUsers * kMaxTargets;                       // [kUsers * kMaxTargets] pool tiles holding targets
    float* qs = reinterpret_cast<float*>(tiles + kUsers * kMaxTargets);  // [G * kNews] filter hits: score, news row, query row
    int* qn = reinterpret_cast<int*>(qs + G * kNews);
    int* qr = qn + G * kNews;
    uint64_t* full = reinterpret_cast<uint64_t*>(qr + G * kNews);
    uint64_t* empty = full + kStages;
    float* lo_s = reinterpret_cast<float*>(empty + kStages);        // [G] per row: its last target in output order
    int* lo_r = reinterpret_cast<int*>(lo_s + G);
    int* tm = lo_r + G;                                             // [G] targets of the row, -1: bad row
    int* n_pro = tm + G;
    int* qc = n_pro + 1;                                            // [2] queue length, by tile parity
    int* rlo = qc + 2;                                              // [G] the row's news range (row_range)
    int* rhi = rlo + G;
    int* iv = rhi + G;                                              // [4] tile_interval
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long q0 = static_cast<long long>(blockIdx.x) * G;
    const int here = static_cast<int>(min(static_cast<long long>(G), p.n_rows - q0));
    const int split = blockIdx.y;

    Ring ring{base, full, empty};
    if (o.P > 1 && warp == 4 && lane == 0) ring_init(ring, &tmAh, &tmAl, &tmNh, &tmNl);
    for (int i = threadIdx.x; i < G * kFiltWords; i += kThreads) filt[i] = 0;
    if (threadIdx.x < 2) qc[threadIdx.x] = 0;
    arch_stage_users(o, q0, here, Ys, w2s);
    __syncthreads();
    // ---- the rows' targets and the membership filter of targets and exclusions ----
    int m = 0, lo = 0, hi = 0;
    if (threadIdx.x < G) {
        const int r = threadIdx.x;
        if (r < here) {
            const long long q = q0 + r, a = p.tgt_offsets[q], cnt = p.tgt_offsets[q + 1] - a;
            const bool ok = row_range(p.row_lo, p.row_hi, q, p.n_news, p.bad_row_flag, lo, hi);
            if (cnt > kMaxTargets) {
                m = -1;
                atomicOr(p.target_flag, 1);
            } else if (!ok) {
                m = -1;
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
        rlo[r] = lo;
        rhi[r] = hi;
    }
    if (p.row_lo != nullptr && threadIdx.x < kUsers) tile_interval(lo, hi, m > 0, iv);
    if (p.excl_offsets != nullptr) {
        bool bad = false;
        for (int r = 0; r < here; ++r)
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
            for (int r = 0; r < G; ++r)
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
    int t0, t1;
    split_tiles(iv, p.row_lo != nullptr, p.tiles, split, p.splits, t0, t1);

    if (warp == 4) {
        // ===================== TMA producer (P > 1): the target tiles, then the split's tiles =====================
        if (o.P > 1 && elect_one()) {
            const int a0 = static_cast<int>(q0 * o.P);
            for (int i = 0; i < npro; ++i) produce_tile(ring, &tmAh, &tmAl, &tmNh, &tmNl, a0, tiles[i], p.k_chunks);
            for (int t = t0; t < t1; ++t) produce_tile(ring, &tmAh, &tmAl, &tmNh, &tmNl, a0, t, p.k_chunks);
        }
        return;
    }

    // ===================== consumer warpgroup =====================
    // prologue: the target scores, from the score tiles of the tiles that hold them (user g's scores in T's row g P)
    for (int i = 0; i < npro; ++i) {
        const int t = tiles[i];
        arch_stage_tile(ring, o, t, p.n_news, p.k_chunks, T, Xs);
        asm volatile("bar.sync 1, 128;" ::: "memory");
        arch_tile_pairs(o, T, Xs, Ys, w2s, Ws, here, [&](int g, int c, float s) { T[g * o.P * kArchTileLd + c] = s; });
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (threadIdx.x < here) {
            const int r = threadIdx.x;
            for (int j = 0; j < tm[r]; ++j) {
                const int col = tr[r * kMaxTargets + j] - t * kNews;
                if (col >= 0 && col < kNews) ts[r * kMaxTargets + j] = T[r * o.P * kArchTileLd + col];
            }
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    // each row's targets into output order (score descending, row ascending); counts start at zero
    bool bad_score = false;
    if (threadIdx.x < G) {
        const int r = threadIdx.x, m = tm[r];
        float* s = ts + r * kMaxTargets;
        int* n = tr + r * kMaxTargets;
        int* ord = tp + r * kMaxTargets;
        for (int j = 0; j < m; ++j) bad_score |= !(fabsf(s[j]) <= 3.402823466e38f);
        for (int j = 1; j < m; ++j) {
            const float sj = s[j];
            const int nj = n[j], oj = ord[j];
            int i = j;
            for (; i > 0 && before(sj, nj, s[i - 1], n[i - 1]); --i) {
                s[i] = s[i - 1];
                n[i] = n[i - 1];
                ord[i] = ord[i - 1];
            }
            s[i] = sj;
            n[i] = nj;
            ord[i] = oj;
        }
        for (int j = 0; j < kMaxTargets; ++j) hist[r * kMaxTargets + j] = 0;
        // threshold: a score counts when it comes before the row's last target
        lo_s[r] = m > 0 ? s[m - 1] : INFINITY;  // nothing comes before (+inf, -1)
        lo_r[r] = m > 0 ? n[m - 1] : -1;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    for (int t = t0; t < t1; ++t) {
        arch_stage_tile(ring, o, t, p.n_news, p.k_chunks, T, Xs);
        asm volatile("bar.sync 1, 128;" ::: "memory");
        arch_tile_pairs(o, T, Xs, Ys, w2s, Ws, here, [&](int g, int c, float s) {
            const int n = t * kNews + c;
            if (lo_r[g] < 0 || n < rlo[g] || n >= rhi[g]) return;  // no target, a bad row, or outside the row's range
            bad_score |= !(fabsf(s) <= 3.402823466e38f);
            if (!before(s, n, lo_s[g], lo_r[g])) return;
            if ((filt[g * kFiltWords + (t & (kFiltWords - 1))] >> c) & 1ull) {  // maybe a target or an exclusion of the row: queued
                const int k = atomicAdd(&qc[t & 1], 1);
                qs[k] = s;
                qn[k] = n;
                qr[k] = g;
                return;
            }
            int b = 0;  // the first target it comes before: exists, the last one
            while (!before(s, n, ts[g * kMaxTargets + b], tr[g * kMaxTargets + b])) ++b;
            atomicAdd(&hist[g * kMaxTargets + b], 1);
        });
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
    // ---- rank of the b-th target in output order: the counts of bins 0 .. b ----
    if (threadIdx.x < here) {
        const int r = threadIdx.x, m = tm[r];
        const long long q = q0 + r;
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

// the top-k kernel and, with several splits, the merge: plain or capped (the instantiation's own profile names)
template <bool kCapped>
static int topk_launch(const CUtensorMap (&tm)[4], const topk::Params& p, cudaStream_t stream) {
    using namespace topk;
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(topk_dot_kernel<kCapped>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmem)));
        attr_set = true;
    }
    const long long user_tiles = (p.n_users + kUsers - 1) / kUsers;
    {
        ProfScope ps(kCapped ? "topk_dot_capped" : "topk_dot", static_cast<int>(p.n_users), p.n_news, p.k, stream);
        topk_dot_kernel<kCapped><<<dim3(static_cast<unsigned>(user_tiles), p.splits), kThreads, kSmem, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    if (p.splits > 1) {
        ProfScope ps(kCapped ? "topk_merge_capped" : "topk_merge", static_cast<int>(p.n_users), p.splits, p.k, stream);
        topk_merge_kernel<kCapped><<<static_cast<unsigned>((p.n_users + kMergeWarps - 1) / kMergeWarps), kMergeWarps * 32, 0, stream>>>(p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

int topk_dot(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D, int k,
             const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category,
             const long long* row_lo, const long long* row_hi, long long* idx, float* score, int* bad_row_flag,
             int* bad_score_flag, void* workspace, long long workspace_bytes, cudaStream_t stream) {
    using namespace topk;
    NR_PROPAGATE(topk_check(n_users, n_news, D, k));
    NR_REQUIRE(ld_users >= D && ld_news >= D, "nr_topk_dot: pitches ld_users=%d ld_news=%d below D=%d", ld_users, ld_news, D);
    NR_REQUIRE((excl_offsets == nullptr) == (excl_rows == nullptr), "nr_topk_dot: excl_offsets and excl_rows go together");
    NR_REQUIRE((row_lo == nullptr) == (row_hi == nullptr), "nr_topk_dot: row_lo and row_hi go together");
    const int splits = topk_splits(n_users, n_news);
    TopkWorkspace ws(workspace, n_users, n_news, D, k, splits);
    NR_REQUIRE(workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && workspace_bytes >= ws.bytes(),
               "nr_topk_dot: workspace of %lld bytes (256-byte aligned) needs %lld", workspace_bytes, ws.bytes());
    if (n_users == 0 || n_news == 0) return 0;
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
    p.cat = categories;
    p.cap = max_per_category;
    p.row_lo = row_lo;
    p.row_hi = row_hi;
    return categories != nullptr ? topk_launch<true>(tm, p, stream) : topk_launch<false>(tm, p, stream);
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
               const long long* row_lo, const long long* row_hi, long long* rank, float* score, int* bad_row_flag,
               int* bad_score_flag, int* target_flag, void* workspace, long long workspace_bytes, cudaStream_t stream) {
    using namespace topk;
    NR_PROPAGATE(pool_ranks_check(n_rows, n_news, D));
    NR_REQUIRE(ld_queries >= D && ld_news >= D, "nr_pool_ranks: pitches ld_queries=%d ld_news=%d below D=%d", ld_queries, ld_news, D);
    NR_REQUIRE((excl_offsets == nullptr) == (excl_rows == nullptr), "nr_pool_ranks: excl_offsets and excl_rows go together");
    NR_REQUIRE((row_lo == nullptr) == (row_hi == nullptr), "nr_pool_ranks: row_lo and row_hi go together");
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
    p.row_lo = row_lo;
    p.row_hi = row_hi;
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

static topk::GramRows gram_rows(const float* news, int ld_news, int D) {
    topk::GramRows g;
    g.news = news;
    g.ld = ld_news;
    g.D = D;
    g.k_chunks = ceil_div(D, 64);
    g.vec4 = ld_news % 4 == 0 && (reinterpret_cast<uintptr_t>(news) & 15) == 0;
    return g;
}

int mmr_rerank(const float* news, long long n_news, int ld_news, int D, const long long* sl_idx, const float* sl_score,
               long long n_users, int depth, int k, float lambda, long long* idx, float* score, int* bad_row_flag,
               cudaStream_t stream) {
    using namespace topk;
    NR_REQUIRE(D >= 1 && D <= 4096, "nr_mmr_rerank: D=%d outside [1, 4096]", D);
    NR_REQUIRE(ld_news >= D, "nr_mmr_rerank: pitch ld_news=%d below D=%d", ld_news, D);
    NR_REQUIRE(n_news >= 0 && n_news < (1ll << 31) - kNews, "nr_mmr_rerank: n_news=%lld outside [0, 2^31 - 64)", n_news);
    NR_REQUIRE(n_users >= 0 && n_users < (1ll << 31) - kUsers, "nr_mmr_rerank: n_users=%lld outside [0, 2^31 - 64)", n_users);
    NR_REQUIRE(depth >= 1 && depth <= kMmrDepth, "nr_mmr_rerank: depth=%d outside [1, %d]", depth, kMmrDepth);
    NR_REQUIRE(k >= 1 && k <= depth, "nr_mmr_rerank: k=%d outside [1, depth=%d]", k, depth);
    NR_REQUIRE(lambda >= 0.f && lambda <= 1.f, "nr_mmr_rerank: lambda=%g outside [0, 1]", static_cast<double>(lambda));
    if (n_users == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(mmr_rerank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kMmrSmem)));
        attr_set = true;
    }
    MmrParams p;
    p.src = gram_rows(news, ld_news, D);
    p.n_news = n_news;
    p.n_users = n_users;
    p.depth = depth;
    p.k = k;
    p.lam = lambda;
    p.one_minus_lam = 1.f - lambda;
    p.sl_idx = sl_idx;
    p.sl_score = sl_score;
    p.idx = idx;
    p.score = score;
    p.bad_row_flag = bad_row_flag;
    ProfScope ps("mmr_rerank", static_cast<int>(n_users), depth, k, stream);
    mmr_rerank_kernel<<<static_cast<unsigned>(n_users), kMmrThreads, kMmrSmem, stream>>>(p);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int list_stats(const float* news, long long n_news, int ld_news, int D, const long long* idx, long long n_rows, int k,
               const int* categories, const int* ks, int n_ks, double* pair_sum, int* distinct, int* bad_row_flag,
               cudaStream_t stream) {
    using namespace topk;
    NR_REQUIRE(D >= 1 && D <= 4096, "nr_list_stats: D=%d outside [1, 4096]", D);
    NR_REQUIRE(ld_news >= D, "nr_list_stats: pitch ld_news=%d below D=%d", ld_news, D);
    NR_REQUIRE(k >= 1 && k <= kMmrDepth, "nr_list_stats: k=%d outside [1, %d]", k, kMmrDepth);
    NR_REQUIRE(n_news >= 0 && n_news < (1ll << 31) - kNews, "nr_list_stats: n_news=%lld outside [0, 2^31 - 64)", n_news);
    NR_REQUIRE(n_rows >= 0 && n_rows < (1ll << 31) - kUsers, "nr_list_stats: n_rows=%lld outside [0, 2^31 - 64)", n_rows);
    NR_REQUIRE(n_ks >= 1 && n_ks <= kListMaxKs, "nr_list_stats: n_ks=%d outside [1, %d]", n_ks, kListMaxKs);
    for (int c = 0; c < n_ks; ++c)
        NR_REQUIRE(ks[c] >= 1 && ks[c] <= k && (c == 0 || ks[c] > ks[c - 1]),
                   "nr_list_stats: ks[%d]=%d is not above the previous cut-off or outside [1, k=%d]", c, ks[c], k);
    NR_REQUIRE((categories == nullptr) == (distinct == nullptr), "nr_list_stats: categories and distinct go together");
    if (n_rows == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(list_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kMmrSmem)));
        attr_set = true;
    }
    ListStatsParams p;
    p.src = gram_rows(news, ld_news, D);
    p.n_news = n_news;
    p.idx = idx;
    p.categories = categories;
    p.k = k;
    p.n_ks = n_ks;
    p.k_max = ks[n_ks - 1];
    for (int c = 0; c < kListMaxKs; ++c) p.ks[c] = c < n_ks ? ks[c] : k;
    p.pair_sum = pair_sum;
    p.distinct = distinct;
    p.bad_row_flag = bad_row_flag;
    ProfScope ps("list_stats", static_cast<int>(n_rows), k, n_ks, stream);
    list_stats_kernel<<<static_cast<unsigned>(n_rows), kMmrThreads, kMmrSmem, stream>>>(p);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---- the archive DNN scorer over the pool ----
static int archive_check(const char* who, long long n_users, int P, long long n_news, long long min_news, int F, int hidden) {
    NR_REQUIRE(P >= 1 && P <= topk::kArchMaxP, "%s: P=%d outside [1, 32]", who, P);
    NR_REQUIRE(hidden >= 1 && hidden <= topk::kArchMaxHid, "%s: hidden=%d outside [1, 32]", who, hidden);
    NR_REQUIRE(F >= 1 && F <= 4096, "%s: F=%d outside [1, 4096]", who, F);
    NR_REQUIRE(n_users >= 0 && n_users < ((1ll << 31) - topk::kUsers) / P, "%s: n_users=%lld x P=%d outside [0, 2^31 - 64)", who,
               n_users, P);
    NR_REQUIRE(n_news >= min_news && n_news < (1ll << 31) - topk::kNews, "%s: n_news=%lld outside [%lld, 2^31 - 64)", who, n_news,
               min_news);
    return 0;
}

// the planes of the archive rows and the news (P > 1 only: P = 1 needs no logits), X and Y
struct ArchPlanes {
    DotPlanes planes;
    float *X, *Y;
    ArchPlanes(WorkspaceLayout& ws, long long n_users, int P, long long n_news, int F, int hidden)
        : planes(ws, P > 1 ? n_users * P : 0, P > 1 ? n_news : 0, F) {
        const int hp = round_up(hidden, 8);
        X = ws.take<float>(n_news * hp);
        Y = ws.take<float>(n_users * P * hp);
    }
    // the TMA maps and planes (P > 1), then X and Y; fills o
    int prepare(const float* archive, long long n_users, int P, const float* news, long long n_news, int F, const float* W1,
                const float* b1, int hidden, const float* w2, const float* b2, CUtensorMap (&tm)[4], topk::ArchOperands& o,
                cudaStream_t stream) const {
        o.P = P;
        o.G = topk::kUsers / P;
        o.hid = hidden;
        o.hp = round_up(hidden, 8);
        o.X = X;
        o.Y = Y;
        o.w2 = w2;
        o.b2 = b2;
        if (P > 1) NR_PROPAGATE(planes.prepare(archive, n_users * P, F, news, n_news, F, F, tm, stream));
        const struct { const float* src; long long rows; int col0; const float* b; float* out; } jobs[2] = {
            {news, n_news, 0, b1, X}, {archive, n_users * P, F, nullptr, Y}};
        for (const auto& j : jobs) {
            if (j.rows == 0) continue;
            ProfScope ps("archive_project", static_cast<int>(j.rows), F, hidden, stream);
            topk::arch_project_kernel<<<static_cast<unsigned>((j.rows + 7) / 8), 256, 0, stream>>>(j.src, j.rows, F, W1 + j.col0, 2 * F,
                                                                                                     j.b, hidden, o.hp, j.out);
            ++g_launches;
            NR_CHECK_CUDA(cudaGetLastError());
        }
        return 0;
    }
};

static int archive_ctas(long long n_users, int P) { return static_cast<int>((n_users + topk::kUsers / P - 1) / (topk::kUsers / P)); }

struct TopkArchiveWorkspace : WorkspaceLayout {
    ArchPlanes ops;
    float* part_score;
    int* part_row;
    TopkArchiveWorkspace(void* base, long long n_users, int P, long long n_news, int F, int hidden, int k, int splits)
        : WorkspaceLayout{static_cast<char*>(base)}, ops(*this, n_users, P, n_news, F, hidden) {
        part_score = take<float>(splits > 1 ? n_users * splits * k : 0);
        part_row = take<int>(splits > 1 ? n_users * splits * k : 0);
    }
};

static int topk_archive_check(long long n_users, int P, long long n_news, int F, int hidden, int k) {
    NR_REQUIRE(k >= 1 && k <= 128, "nr_topk_archive: k=%d outside [1, 128]", k);
    return archive_check("nr_topk_archive", n_users, P, n_news, 0, F, hidden);
}

static int archive_splits(long long n_users, int P, long long n_news) {
    return topk_splits(static_cast<long long>(archive_ctas(n_users, P)) * topk::kUsers, n_news);
}

long long topk_archive_workspace(long long n_users, int P, long long n_news, int F, int hidden, int k) {
    if (topk_archive_check(n_users, P, n_news, F, hidden, k) != 0) return -1;
    return TopkArchiveWorkspace(nullptr, n_users, P, n_news, F, hidden, k, archive_splits(n_users, P, n_news)).bytes();
}

template <bool kCapped>
static int topk_archive_launch(const CUtensorMap (&tm)[4], const topk::Params& p, const topk::ArchOperands& o, cudaStream_t stream) {
    using namespace topk;
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(topk_archive_kernel<kCapped>, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
        attr_set = true;
    }
    const size_t smem = 1024 + ArchSmem(o.P, o.G, o.hp, topk_archive_rest(o.G)).bytes;
    {
        ProfScope ps(kCapped ? "topk_archive_capped" : "topk_archive", static_cast<int>(p.n_users), p.n_news, p.k, stream);
        topk_archive_kernel<kCapped><<<dim3(static_cast<unsigned>(archive_ctas(p.n_users, o.P)), p.splits), kThreads, smem, stream>>>(
            tm[0], tm[1], tm[2], tm[3], p, o);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    if (p.splits > 1) {
        ProfScope ps(kCapped ? "topk_merge_capped" : "topk_merge", static_cast<int>(p.n_users), p.splits, p.k, stream);
        topk_merge_kernel<kCapped><<<static_cast<unsigned>((p.n_users + kMergeWarps - 1) / kMergeWarps), kMergeWarps * 32, 0, stream>>>(p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

int topk_archive(const float* archive, long long n_users, int P, const float* news, long long n_news, int F, const float* W1,
                 const float* b1, int hidden, const float* w2, const float* b2, int k, const long long* excl_offsets,
                 const long long* excl_rows, const int* categories, int max_per_category, const long long* row_lo,
                 const long long* row_hi, long long* idx, float* score, int* bad_row_flag, int* bad_score_flag, void* workspace,
                 long long workspace_bytes, cudaStream_t stream) {
    using namespace topk;
    NR_PROPAGATE(topk_archive_check(n_users, P, n_news, F, hidden, k));
    NR_REQUIRE((excl_offsets == nullptr) == (excl_rows == nullptr), "nr_topk_archive: excl_offsets and excl_rows go together");
    NR_REQUIRE(categories == nullptr || max_per_category >= 1, "nr_topk_archive: max_per_category=%d below 1", max_per_category);
    NR_REQUIRE((row_lo == nullptr) == (row_hi == nullptr), "nr_topk_archive: row_lo and row_hi go together");
    const int splits = archive_splits(n_users, P, n_news);
    TopkArchiveWorkspace ws(workspace, n_users, P, n_news, F, hidden, k, splits);
    NR_REQUIRE(workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && workspace_bytes >= ws.bytes(),
               "nr_topk_archive: workspace of %lld bytes (256-byte aligned) needs %lld", workspace_bytes, ws.bytes());
    if (n_users == 0 || n_news == 0) return 0;
    CUtensorMap tm[4] = {};
    ArchOperands o;
    NR_PROPAGATE(ws.ops.prepare(archive, n_users, P, news, n_news, F, W1, b1, hidden, w2, b2, tm, o, stream));
    Params p;
    p.n_users = n_users;
    p.n_news = static_cast<int>(n_news);
    p.k = k;
    p.k_chunks = ceil_div(F, 64);
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
    p.cat = categories;
    p.cap = max_per_category;
    p.row_lo = row_lo;
    p.row_hi = row_hi;
    return categories != nullptr ? topk_archive_launch<true>(tm, p, o, stream) : topk_archive_launch<false>(tm, p, o, stream);
}

struct RankArchiveWorkspace : WorkspaceLayout {
    ArchPlanes ops;
    int* part;
    RankArchiveWorkspace(void* base, long long n_rows, int P, long long n_news, int F, int hidden, int splits)
        : WorkspaceLayout{static_cast<char*>(base)}, ops(*this, n_rows, P, n_news, F, hidden) {
        part = take<int>(splits > 1 ? n_rows * splits * topk::kMaxTargets : 0);
    }
};

long long pool_ranks_archive_workspace(long long n_rows, int P, long long n_news, int F, int hidden) {
    if (archive_check("nr_pool_ranks_archive", n_rows, P, n_news, 1, F, hidden) != 0) return -1;
    return RankArchiveWorkspace(nullptr, n_rows, P, n_news, F, hidden, archive_splits(n_rows, P, n_news)).bytes();
}

int pool_ranks_archive(const float* archive, long long n_rows, int P, const float* news, long long n_news, int F, const float* W1,
                       const float* b1, int hidden, const float* w2, const float* b2, const long long* tgt_offsets,
                       const long long* tgt_rows, const long long* excl_offsets, const long long* excl_rows,
                       const long long* row_lo, const long long* row_hi, long long* rank, float* score, int* bad_row_flag,
                       int* bad_score_flag, int* target_flag, void* workspace, long long workspace_bytes, cudaStream_t stream) {
    using namespace topk;
    NR_PROPAGATE(archive_check("nr_pool_ranks_archive", n_rows, P, n_news, 1, F, hidden));
    NR_REQUIRE((excl_offsets == nullptr) == (excl_rows == nullptr), "nr_pool_ranks_archive: excl_offsets and excl_rows go together");
    NR_REQUIRE((row_lo == nullptr) == (row_hi == nullptr), "nr_pool_ranks_archive: row_lo and row_hi go together");
    const int splits = archive_splits(n_rows, P, n_news);
    RankArchiveWorkspace ws(workspace, n_rows, P, n_news, F, hidden, splits);
    NR_REQUIRE(workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && workspace_bytes >= ws.bytes(),
               "nr_pool_ranks_archive: workspace of %lld bytes (256-byte aligned) needs %lld", workspace_bytes, ws.bytes());
    if (n_rows == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(pool_ranks_archive_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
        attr_set = true;
    }
    CUtensorMap tm[4] = {};
    ArchOperands o;
    NR_PROPAGATE(ws.ops.prepare(archive, n_rows, P, news, n_news, F, W1, b1, hidden, w2, b2, tm, o, stream));
    RankParams p;
    p.n_rows = n_rows;
    p.n_news = static_cast<int>(n_news);
    p.k_chunks = ceil_div(F, 64);
    p.tiles = static_cast<int>((n_news + kNews - 1) / kNews);
    p.splits = splits;
    p.tgt_offsets = tgt_offsets;
    p.tgt_rows = tgt_rows;
    p.excl_offsets = excl_offsets;
    p.excl_rows = excl_rows;
    p.row_lo = row_lo;
    p.row_hi = row_hi;
    p.rank = rank;
    p.score = score;
    p.part = ws.part;
    p.bad_row_flag = bad_row_flag;
    p.bad_score_flag = bad_score_flag;
    p.target_flag = target_flag;
    const size_t smem = 1024 + ArchSmem(o.P, o.G, o.hp, ranks_archive_rest(o.G)).bytes;
    {
        ProfScope ps("pool_ranks_archive", static_cast<int>(n_rows), static_cast<int>(n_news), splits, stream);
        pool_ranks_archive_kernel<<<dim3(static_cast<unsigned>(archive_ctas(n_rows, P)), splits), kThreads, smem, stream>>>(
            tm[0], tm[1], tm[2], tm[3], p, o);
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

// the largest shared memory either archive kernel asks for, over every P (G = 64 / P users per CTA)
static constexpr int archive_smem_max() {
    int m = 0;
    for (int P = 1; P <= topk::kArchMaxP; ++P) {
        const int G = topk::kUsers / P;
        const int a = topk::ArchSmem(P, G, topk::kArchMaxHid, topk::topk_archive_rest(G)).bytes;
        const int b = topk::ArchSmem(P, G, topk::kArchMaxHid, topk::ranks_archive_rest(G)).bytes;
        m = std::max(m, std::max(a, b));
    }
    return 1024 + m;
}
static_assert(archive_smem_max() <= 232448, "topk_archive_kernel / pool_ranks_archive_kernel: shared memory");

}  // namespace nr
