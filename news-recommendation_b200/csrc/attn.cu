// Multi-head self-attention core (reference src/model/general/attention/multihead_self.py:15-23) on the
// legacy tensor path (mma.sync m16n8k16 bf16 + ldmatrix): the per-(sequence, head) products are 20x20x20 /
// 50x50x20 -- 3 % of the model's FLOPs and far too small for a 128-row wgmma tile -- so one WARP owns one
// head, all operands live in shared-memory tiles and nothing but Q|K|V (+dCtx) is read from HBM.
//
//   forward : S = QK^T/sqrt(dk);  A = exp(S)/(sum exp(S) + 1e-8)  [stable form];  ctx = A V
//   backward: dA = dCtx V^T;  dS = A (dA - sum A dA)/sqrt(dk);  dQ = dS K;  dK = dS^T Q;  dV = A^T dCtx
//
// bf16 storage contract (mirrored by the oracle): A and dS are rounded to bf16 as tensor-core operands,
// all softmax arithmetic is fp32.
#include <algorithm>

#include "nr_common.cuh"
#include "nr_mma.cuh"
#include "nr_ops.h"

namespace nr {

namespace {

using namespace mma;

constexpr int kPitch = 40;   // bf16 elements per tile row (80 B: 16-byte aligned, ldmatrix conflict-free), generic kernels
constexpr int kPitch24 = 24; // fixed-shape d_k = 20 kernels: 48-byte rows (also conflict-free: 8 rows x 16 B hit 8 distinct bank
                             // quads); the second k-step over d_k is then an m16n8k8 MMA over columns 16..23 (20..23 stay zero).
                             // 40 % less shared memory per tile -> 4 instead of 3 resident CTAs (backward), 6 instead of 5 (forward):
                             // the kernels are latency bound (25-36 % issue-active under ncu), residency is what they lack.
constexpr int kWarps = 4;    // warps per CTA
constexpr int kStages = 2;   // tasks in flight per copy ring
// Rows of a tile: 32 for the per-warp kernels (T <= 32), 64 for the cooperative ones (32 < T <= 64).
__host__ __device__ constexpr int tile_rows(bool coop) { return coop ? 64 : 32; }
// The reference's head shape (config.py: 15 heads x 20), at the sequence length each schedule sees in the reference:
// 20 title words (per-warp kernels, dense-section callers) and 50 clicked news (cooperative kernels, user encoder).
constexpr int kFixedDk = 20, kFixedHeads = 15;
__host__ __device__ constexpr int fixed_T(bool coop) { return coop ? 50 : 20; }

// A fragment (16 x 16) of a row-major [row][k] tile:           rows row0.., k columns k0..
__device__ __forceinline__ void load_a(uint32_t* a, const __nv_bfloat16* tile, int pitch, int row0, int k0, int lane) {
    ldsm_x4(a, tile + (row0 + (lane & 15)) * pitch + k0 + ((lane >> 4) << 3));
}
// 16 x 8 A fragment / 8 x 8 B fragment (B[k][n] = tile[n][k]) of the m16n8k8 tail step
__device__ __forceinline__ void load_a8(uint32_t* a, const __nv_bfloat16* tile, int pitch, int row0, int k0, int lane) {
    ldsm_x2(a, tile + (row0 + (lane & 15)) * pitch + k0);
}
__device__ __forceinline__ void load_b8(uint32_t* b, const __nv_bfloat16* tile, int pitch, int n0, int k0, int lane) {
    ldsm_x1(b, tile + (n0 + (lane & 7)) * pitch + k0);
}
// A fragment of A = M^T where M is stored row-major [k][m]:      m rows m0.., k columns k0..
__device__ __forceinline__ void load_a_t(uint32_t* a, const __nv_bfloat16* tile, int pitch, int m0, int k0, int lane) {
    ldsm_x4_t(a, tile + (k0 + (lane & 7) + ((lane >> 4) << 3)) * pitch + m0 + (((lane >> 3) & 1) << 3));
}
// B fragment (k16 x n8) with B[k][n] = tile[n][k] (tile row-major [n][k]):   n rows n0.., k columns k0..
__device__ __forceinline__ void load_b(uint32_t* b, const __nv_bfloat16* tile, int pitch, int n0, int k0, int lane) {
    ldsm_x2(b, tile + (n0 + (lane & 7)) * pitch + k0 + (((lane >> 3) & 1) << 3));
}
// B fragment with B[k][n] = tile[k][n] (tile row-major [k][n]):                k rows k0.., n columns n0..
__device__ __forceinline__ void load_b_t(uint32_t* b, const __nv_bfloat16* tile, int pitch, int k0, int n0, int lane) {
    ldsm_x2_t(b, tile + (k0 + (lane & 7) + (((lane >> 3) & 1) << 3)) * pitch + n0);
}

// Row-block softmax on the S fragments of one 16-row m-tile.  s[nt][4] holds (row g: c0,c1 ; row g+8: c2,c3)
// for key columns nt*8 + 2t, +1.  Input scores are pre-scaled into the log2 domain.  Returns P in place.
template <int NTJ>
__device__ __forceinline__ void softmax_rows(float (*s)[4], int T, int t4, int ntj, float sc, bool dead1 = false) {
    // raw scores in, probabilities out; `sc` = log2(e)/sqrt(d_k) is folded into the exp2 argument.
    // Only the last live n-tile can contain key columns >= T; tiles >= ntj are dead (skipped everywhere).
    // dead1: rows g+8 of this 16-row block are all >= T (compile-time for the fixed shapes): their probabilities are
    // forced to zero without computing anything (for T = 20 that is half of the second row block).
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < NTJ; ++nt) {
        if (nt >= ntj) break;
        if (nt * 8 + 8 > T) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const bool ok = nt * 8 + 2 * t4 + e < T;
                s[nt][e] = ok ? s[nt][e] : -INFINITY;
                if (!dead1) s[nt][2 + e] = ok ? s[nt][2 + e] : -INFINITY;
            }
        }
        m0 = fmaxf(m0, fmaxf(s[nt][0], s[nt][1]));
        if (!dead1) m1 = fmaxf(m1, fmaxf(s[nt][2], s[nt][3]));
    }
    m0 = quad_max(m0) * sc;
    if (!dead1) m1 = quad_max(m1) * sc;
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < NTJ; ++nt) {
        if (nt >= ntj) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; continue; }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            s[nt][e] = exp2f(fmaf(s[nt][e], sc, -m0));
            l0 += s[nt][e];
            if (!dead1) {
                s[nt][2 + e] = exp2f(fmaf(s[nt][2 + e], sc, -m1));
                l1 += s[nt][2 + e];
            } else {
                s[nt][2 + e] = 0.f;
            }
        }
    }
    l0 = quad_sum(l0);
    const float i0 = 1.f / (l0 + 1e-8f * exp2f(-m0));  // == exp(S)/(sum exp(S) + 1e-8) of the reference
    float i1 = 0.f;
    if (!dead1) {
        l1 = quad_sum(l1);
        i1 = 1.f / (l1 + 1e-8f * exp2f(-m1));
    }
#pragma unroll
    for (int nt = 0; nt < NTJ; ++nt) {
        if (nt >= ntj) break;
        s[nt][0] *= i0;
        s[nt][1] *= i0;
        if (!dead1) {
            s[nt][2] *= i1;
            s[nt][3] *= i1;
        }
    }
}


// ------------------------------------------------------------------------------------------------
// Warp-private task pipeline.  A task is one (sequence, head); a warp walks tasks gw, gw+W, gw+2W, ... and keeps
// kStages of them in flight with cp.async (8-byte pieces when d_k % 4 == 0, 4-byte when even, else plain
// 2-byte copies), so that ~40-60 KB per SM are always outstanding -- the first (CTA-staged, synchronous)
// version of this kernel was latency bound at ~270 GB/s.
// Tile = [TP rows][kPitch] bf16, valid region [T][dk]; everything outside stays zero for the whole kernel.
// ------------------------------------------------------------------------------------------------

__device__ __forceinline__ void cp_async8(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// global rows [T][dk] at g (pitch ld, elements)  ->  tile rows.  piece = bytes per copy (8 / 4 / 2).
__device__ __forceinline__ void tile_load(__nv_bfloat16* tile, const __nv_bfloat16* g, int ld, int T, int dk, int piece, int lane, int nthr = 32, int pitch = kPitch) {
    const int epp = piece >> 1;        // elements per piece
    const int ppr = dk / epp;          // pieces per row
    const float inv = 1.0f / static_cast<float>(ppr);
    const int n = T * ppr;
    for (int i = lane; i < n; i += nthr) {
        const int r = static_cast<int>((static_cast<float>(i) + 0.5f) * inv);
        const int c = (i - r * ppr) * epp;
        __nv_bfloat16* dst = tile + r * pitch + c;
        const __nv_bfloat16* src = g + static_cast<size_t>(r) * ld + c;
        if (piece == 8) cp_async8(dst, src);
        else if (piece == 4) cp_async4(dst, src);
        else *dst = *src;
    }
}
__device__ __forceinline__ void tile_store(const __nv_bfloat16* tile, __nv_bfloat16* g, int ld, int T, int dk, int piece, int lane, int nthr = 32, int pitch = kPitch) {
    const int epp = piece >> 1;
    const int ppr = dk / epp;
    const float inv = 1.0f / static_cast<float>(ppr);
    const int n = T * ppr;
    for (int i = lane; i < n; i += nthr) {
        const int r = static_cast<int>((static_cast<float>(i) + 0.5f) * inv);
        const int c = (i - r * ppr) * epp;
        const __nv_bfloat16* src = tile + r * pitch + c;
        __nv_bfloat16* dst = g + static_cast<size_t>(r) * ld + c;
        if (piece == 8) *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(src);
        else if (piece == 4) *reinterpret_cast<uint32_t*>(dst) = *reinterpret_cast<const uint32_t*>(src);
        else *dst = *src;
    }
}
// Per-lane copy plan: the (row, column) of every piece a lane moves is the same for every task, so the
// offsets are computed ONCE per kernel (ncu: per-piece index arithmetic was 30 % of all instructions).
constexpr int kMaxP = 4;  // pieces per lane covered by the plan (T * pieces_per_row <= 128); larger tiles use the loops
struct PieceMap {
    int total;        // pieces of the whole tile: lane l moves pieces l, l+32, ... < total
    int lane;
    int n;            // pieces of this lane
    int src[kMaxP];   // element offset in the global matrix:  r * ld + c
    int dst[kMaxP];   // element offset in the tile:            r * kPitch + c
    int row[kMaxP];
    int col[kMaxP];
};
__device__ __forceinline__ bool make_piece_map(PieceMap& m, int T, int dk, int piece, int ld, int lane, int pitch = kPitch) {
    const int epp = piece >> 1, ppr = dk / epp, n = T * ppr;
    m.n = 0;
    m.total = n;
    m.lane = lane;
    if (piece < 4 || n > kMaxP * 32) return false;
#pragma unroll
    for (int k = 0; k < kMaxP; ++k) {
        const int i = lane + 32 * k;
        const int r = i / ppr, c = (i - r * ppr) * epp;
        m.src[k] = r * ld + c;
        m.dst[k] = r * pitch + c;
        m.row[k] = r;
        m.col[k] = c;
        if (i < n) m.n = k + 1;
    }
    return true;
}
__device__ __forceinline__ void tile_load_map(uint32_t tile_saddr, const __nv_bfloat16* g, const PieceMap& m, int piece) {
#pragma unroll
 for (int k = 0; k < kMaxP; ++k) {
        if (m.lane + 32 * k < m.total) {
            if (piece == 8)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(tile_saddr + 2 * m.dst[k]), "l"(g + m.src[k]) : "memory");
            else
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(tile_saddr + 2 * m.dst[k]), "l"(g + m.src[k]) : "memory");
        }
    }
}
__device__ __forceinline__ void tile_store_map(const __nv_bfloat16* tile, __nv_bfloat16* g, const PieceMap& m, int piece) {
#pragma unroll
    for (int k = 0; k < kMaxP; ++k) {
        if (m.lane + 32 * k < m.total) {
            if (piece == 8) *reinterpret_cast<uint2*>(g + m.src[k]) = *reinterpret_cast<const uint2*>(tile + m.dst[k]);
            else *reinterpret_cast<uint32_t*>(g + m.src[k]) = *reinterpret_cast<const uint32_t*>(tile + m.dst[k]);
        }
    }
}
// context tile -> global with dropout (one counter hash per 4 aligned columns), offsets from the plan
__device__ __forceinline__ void tile_store_dropout_map(const __nv_bfloat16* tile, __nv_bfloat16* g, const PieceMap& m, int piece, int ld,
                                                       long long row0, int col0, const Dropout& drop) {
#pragma unroll
    for (int k = 0; k < kMaxP; ++k) {
        if (m.lane + 32 * k < m.total) {
            const long long row = row0 + m.row[k];
            const int gc = col0 + m.col[k];
            if (piece == 8) {
                float mk[4];
                drop.mask4(row, ld, gc, mk);
                const uint2 u = *reinterpret_cast<const uint2*>(tile + m.dst[k]);
                const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
                *reinterpret_cast<uint2*>(g + m.src[k]) = make_uint2(pack_bf16x2(a.x * mk[0], a.y * mk[1]), pack_bf16x2(b.x * mk[2], b.y * mk[3]));
            } else {
                const float2 mk = drop.mask2(row, ld, gc);
                const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(tile + m.dst[k]));
                *reinterpret_cast<uint32_t*>(g + m.src[k]) = pack_bf16x2(a.x * mk.x, a.y * mk.y);
            }
        }
    }
}

// context tile -> global with the dropout mask applied on the fly (one counter hash per 4 aligned columns)
__device__ __forceinline__ void tile_store_dropout(const __nv_bfloat16* tile, __nv_bfloat16* g, int ld, int T, int dk, int piece, int lane,
                                                   long long row0, int col0, const Dropout& drop, int nthr = 32, int pitch = kPitch) {
    const int epp = piece >> 1;
    const int ppr = dk / epp;
    const float inv = 1.0f / static_cast<float>(ppr);
    const int n = T * ppr;
    for (int i = lane; i < n; i += nthr) {
        const int r = static_cast<int>((static_cast<float>(i) + 0.5f) * inv);
        const int c = (i - r * ppr) * epp;
        const __nv_bfloat16* src = tile + r * pitch + c;
        __nv_bfloat16* dst = g + static_cast<size_t>(r) * ld + c;
        const int gc = col0 + c;
        if (piece == 8) {
            float mk[4];
            drop.mask4(row0 + r, ld, gc, mk);
            const uint2 u = *reinterpret_cast<const uint2*>(src);
            const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
            *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(a.x * mk[0], a.y * mk[1]), pack_bf16x2(b.x * mk[2], b.y * mk[3]));
        } else if (piece == 4) {
            const float2 mk = drop.mask2(row0 + r, ld, gc);
            const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(src));
            *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(a.x * mk.x, a.y * mk.y);
        } else {
            *dst = __float2bfloat16_rn(__bfloat162float(*src) * drop.mask2(row0 + r, ld, gc).x);
        }
    }
}
__host__ __device__ inline int piece_bytes(int dk, int ld_a, int ld_b, int d) {
    if ((dk % 4) == 0 && (ld_a % 4) == 0 && (ld_b % 4) == 0 && (d % 4) == 0) return 8;
    if ((dk % 2) == 0 && (ld_a % 2) == 0 && (ld_b % 2) == 0 && (d % 2) == 0) return 4;
    return 2;
}
// the backward also stores dQ | dK | dV rows of pitch ld_out in pieces
__host__ __device__ inline int piece_bytes_bwd(int dk, int ld_a, int ld_b, int d, int ld_out) {
    const int piece = piece_bytes(dk, ld_a, ld_b, d);
    return (piece == 8 && (ld_out % 4) == 0) ? 8 : ((piece >= 4 && (ld_out % 2) == 0) ? 4 : 2);
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
// Template parameters:
//   NTD   8-column n-tiles over d_k (2: d_k <= 16, 3: <= 24, 4: <= 32); KSD = 16-wide k-steps over d_k.
//   FAST  per-lane copy plans (PieceMap) instead of the copy loops.
//   FIXED the reference's head shape (T = fixed_T(COOP), d_k 20, 15 heads) at compile time (8-byte pieces guaranteed by
//         the launcher): every shape guard, the piece plan and the task -> (sequence, head) division fold away.  ncu on
//         the run-time shaped kernel: 1200 warp instructions per 20x20 head, 650 of them integer/predicate/branch overhead.
//   COOP  history-level attention (T > 32): the kWarps = TP/16 warps of a CTA share ONE task -- warp w owns the 16-row
//         block w -- instead of walking private tasks: 512 sequences x 15 heads are only 7,680 tasks, and one warp per
//         50x50 head left 3 warps per SM resident (0.28 ms for 4 % of the tokens).  Tiles are loaded/stored by all
//         threads, phases are separated by __syncthreads instead of __syncwarp.
template <int NTD, bool FAST, bool FIXED, bool COOP>
__global__ void __launch_bounds__(kWarps * 32, COOP ? 3 : (FIXED ? 8 : 5)) mhsa_mma_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, int ld, int sec, long long n_seq,
                                                                  int T_, int heads_, int dk_, __nv_bfloat16* __restrict__ ctx,
                                                                  int ld_ctx, Dropout drop) {
    constexpr int TP = tile_rows(COOP), NTJ = TP / 8, MT = TP / 16, KSD = (NTD + 1) / 2;
    constexpr int CT = FIXED ? fixed_T(COOP) : 0;
    constexpr int PT = FIXED ? kPitch24 : kPitch;  // tile row pitch
    constexpr bool K8T = FIXED;                    // last k-step over d_k is an m16n8k8 (columns 16..23)
    constexpr int KS16 = K8T ? KSD - 1 : KSD;
    const int T = FIXED ? CT : T_, heads = FIXED ? kFixedHeads : heads_, dk = FIXED ? kFixedDk : dk_;
    // A tile holds exactly T rows (pitch PT).  Fragment loads of rows >= T run into the neighbouring tile or the
    // zeroed slack behind the last one: finite bytes that only ever meet zero probabilities / unused output rows.
    const int TILE = T * PT;
    extern __shared__ __align__(16) __nv_bfloat16 sm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int d = heads * dk;
    static_assert(!COOP || (kWarps == TP / 16 && !FAST), "cooperative CTAs: one warp per 16-row block, generic copy loops");
    for (int i = tid; i < ((COOP ? 1 : kWarps) * kStages * 3 * TILE + (TP - T) * PT) / 2; i += blockDim.x) reinterpret_cast<uint32_t*>(sm)[i] = 0u;
    __syncthreads();
    __nv_bfloat16* wbase = sm + (COOP ? 0 : warp) * kStages * 3 * TILE;
    const int ctid = COOP ? tid : lane, cnt = COOP ? kWarps * 32 : 32;  // who copies a task's tiles
    auto phase_sync = [&]() { if (COOP) __syncthreads(); else __syncwarp(); };
    const float sc = rsqrtf(static_cast<float>(dk)) * 1.4426950408889634f;
    const int ntj = (T + 7) >> 3;
    const int piece = FIXED ? 8 : piece_bytes(dk, ld, ld_ctx, sec);
    const int n_tasks = static_cast<int>(n_seq * heads);  // < 2^31, checked by the launcher
    const int W = COOP ? gridDim.x : gridDim.x * kWarps;
    const int gw = COOP ? blockIdx.x : blockIdx.x * kWarps + warp;
    PieceMap lmap, smap;
    if (FAST) {
        make_piece_map(lmap, T, dk, piece, ld, lane, PT);
        make_piece_map(smap, T, dk, piece, ld_ctx, lane, PT);
    }
    const uint32_t wbase_s = smem_u32(wbase);

    auto prefetch = [&](int task, int stage) {
        if (task < n_tasks) {
            const int seq = task / heads;
            const int h = task - seq * heads;
            const __nv_bfloat16* src = qkv + static_cast<long long>(seq) * T * ld + h * dk;
            if constexpr (FAST) {
                const uint32_t t0s = wbase_s + 2 * stage * 3 * TILE;
                tile_load_map(t0s, src, lmap, piece);
                tile_load_map(t0s + 2 * TILE, src + sec, lmap, piece);
                tile_load_map(t0s + 4 * TILE, src + 2 * sec, lmap, piece);
            } else {
                __nv_bfloat16* t0 = wbase + stage * 3 * TILE;
                tile_load(t0, src, ld, T, dk, piece, ctid, cnt, PT);
                tile_load(t0 + TILE, src + sec, ld, T, dk, piece, ctid, cnt, PT);
                tile_load(t0 + 2 * TILE, src + 2 * sec, ld, T, dk, piece, ctid, cnt, PT);
            }
        }
        cp_commit();
    };
#pragma unroll
    for (int s0 = 0; s0 < kStages - 1; ++s0) prefetch(gw + s0 * W, s0);

    int stage = 0;
    for (int task = gw; task < n_tasks; task += W) {
        cp_wait<kStages - 2>();
        phase_sync();
        // the stage consumed in the previous iteration is free again: refill it before computing this task
        prefetch(task + (kStages - 1) * W, (stage + kStages - 1) % kStages);
        const long long seq = task / heads;
        const int h = task - static_cast<int>(seq) * heads;
        __nv_bfloat16* q = wbase + stage * 3 * TILE;
        const __nv_bfloat16* k = q + TILE;
        const __nv_bfloat16* v = q + 2 * TILE;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
            if (mt * 16 >= T) break;
            if (COOP && mt != warp) continue;
            float s[NTJ][4];
#pragma unroll
            for (int nt = 0; nt < NTJ; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < KS16; ++ks) {
                uint32_t a[4];
                load_a(a, q, PT, mt * 16, ks * 16, lane);
#pragma unroll
                for (int nt = 0; nt < NTJ; ++nt) {
                    if (nt >= ntj) break;
                    uint32_t b[2];
                    load_b(b, k, PT, nt * 8, ks * 16, lane);
                    mma_bf16(s[nt], a, b);
                }
            }
            if constexpr (K8T) {
                uint32_t a[2];
                load_a8(a, q, PT, mt * 16, KS16 * 16, lane);
#pragma unroll
                for (int nt = 0; nt < NTJ; ++nt) {
                    if (nt >= ntj) break;
                    uint32_t b[1];
                    load_b8(b, k, PT, nt * 8, KS16 * 16, lane);
                    mma_bf16_k8(s[nt], a, b);
                }
            }
            const bool dead1 = FIXED && mt * 16 + 8 >= CT;  // folds after unrolling
            softmax_rows<NTJ>(s, T, t4, ntj, sc, dead1);
            float o[NTD][4];
#pragma unroll
            for (int nd = 0; nd < NTD; ++nd) o[nd][0] = o[nd][1] = o[nd][2] = o[nd][3] = 0.f;
#pragma unroll
            for (int kj = 0; kj < MT; ++kj) {
                if (kj * 16 >= T) break;
                uint32_t a[4];
                a[0] = pack_bf16x2(s[2 * kj][0], s[2 * kj][1]);
                a[1] = pack_bf16x2(s[2 * kj][2], s[2 * kj][3]);
                a[2] = pack_bf16x2(s[2 * kj + 1][0], s[2 * kj + 1][1]);
                a[3] = pack_bf16x2(s[2 * kj + 1][2], s[2 * kj + 1][3]);
#pragma unroll
                for (int nd = 0; nd < NTD; ++nd) {
                    uint32_t b[2];
                    load_b_t(b, v, PT, kj * 16, nd * 8, lane);
                    mma_bf16(o[nd], a, b);
                }
            }
            // context rows replace this m-tile's (now dead) Q rows; only the valid [T][dk] region is touched
            __syncwarp();
#pragma unroll
            for (int nd = 0; nd < NTD; ++nd) {
                const int col = nd * 8 + 2 * t4;
                if (col >= dk) continue;
                const bool pair = col + 1 < dk;
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    if (FIXED && mt * 16 + hf * 8 >= CT) continue;  // whole half-block past T: folds after unrolling
                    const int r = mt * 16 + g + hf * 8;
                    if (r >= T) continue;
                    const float v0 = o[nd][2 * hf], v1 = pair ? o[nd][2 * hf + 1] : 0.f;
                    *reinterpret_cast<uint32_t*>(q + r * PT + col) = pack_bf16x2(v0, v1);
                }
            }
        }
        phase_sync();
        __nv_bfloat16* out = ctx + seq * T * static_cast<long long>(ld_ctx);
        if constexpr (FAST) {
            if (drop.active()) tile_store_dropout_map(q, out + h * dk, smap, piece, ld_ctx, seq * T, h * dk, drop);
            else tile_store_map(q, out + h * dk, smap, piece);
        } else if (drop.active()) {
            tile_store_dropout(q, out + h * dk, ld_ctx, T, dk, piece, ctid, seq * T, h * dk, drop, cnt, PT);
        } else {
            tile_store(q, out + h * dk, ld_ctx, T, dk, piece, ctid, cnt, PT);
        }
        if (h == 0) {  // ones column + zero tail of the padded context rows
            for (int i = ctid; i < T * (ld_ctx - d); i += cnt) {
                const int r = i / (ld_ctx - d), c = i - r * (ld_ctx - d);
                out[static_cast<size_t>(r) * ld_ctx + d + c] = __float2bfloat16_rn(c == 0 ? 1.0f : 0.f);
            }
        }
        phase_sync();
        stage = (stage + 1) % kStages;
    }
    cp_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
template <int NTD, bool FAST, bool FIXED, bool COOP>
__global__ void __launch_bounds__(kWarps * 32, COOP ? 3 : (FIXED ? 4 : 3)) mhsa_mma_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, int ld, int sec,
                                                                  const __nv_bfloat16* __restrict__ dctx, int ld_dctx,
                                                                  long long n_seq, int T_, int heads_, int dk_,
                                                                  __nv_bfloat16* __restrict__ dqkv, int ld_d) {
    constexpr int TP = tile_rows(COOP), NTJ = TP / 8, MT = TP / 16, SP = TP + 8, KSD = (NTD + 1) / 2;
    constexpr int CT = FIXED ? fixed_T(COOP) : 0;
    constexpr int PT = FIXED ? kPitch24 : kPitch;
    constexpr bool K8T = FIXED;
    constexpr int KS16 = K8T ? KSD - 1 : KSD;
    const int T = FIXED ? CT : T_, heads = FIXED ? kFixedHeads : heads_, dk = FIXED ? kFixedDk : dk_;
    const int TILE = T * PT;  // packed rows, see the forward kernel
    extern __shared__ __align__(16) __nv_bfloat16 sm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int d = heads * dk;
    const int PER_WARP = kStages * 4 * TILE + 2 * TP * SP;  // the P/dS scratch behind a warp's tiles doubles as read slack
    static_assert(!COOP || (kWarps == TP / 16 && !FAST), "cooperative CTAs: one warp per 16-row block, generic copy loops");
    for (int i = tid; i < (COOP ? 1 : kWarps) * PER_WARP / 2; i += blockDim.x) reinterpret_cast<uint32_t*>(sm)[i] = 0u;
    __syncthreads();
    __nv_bfloat16* wbase = sm + (COOP ? 0 : warp) * PER_WARP;
    const int ctid = COOP ? tid : lane, cnt = COOP ? kWarps * 32 : 32;
    auto phase_sync = [&]() { if (COOP) __syncthreads(); else __syncwarp(); };
    __nv_bfloat16* ps = wbase + kStages * 4 * TILE;  // [TP][SP] probabilities (bf16)
    __nv_bfloat16* ds = ps + TP * SP;                // [TP][SP] score gradients (bf16)
    const float rs = rsqrtf(static_cast<float>(dk));
    const float sc = rs * 1.4426950408889634f;
    const int ntj = (T + 7) >> 3;
    const int piece = FIXED ? 8 : piece_bytes_bwd(dk, ld, ld_dctx, sec, ld_d);
    const int n_tasks = static_cast<int>(n_seq * heads);
    const int W = COOP ? gridDim.x : gridDim.x * kWarps;
    const int gw = COOP ? blockIdx.x : blockIdx.x * kWarps + warp;
    PieceMap lmap, gmap, smap;
    if (FAST) {
        make_piece_map(lmap, T, dk, piece, ld, lane, PT);
        make_piece_map(gmap, T, dk, piece, ld_dctx, lane, PT);
        make_piece_map(smap, T, dk, piece, ld_d, lane, PT);
    }
    const uint32_t wbase_s = smem_u32(wbase);

    auto prefetch = [&](int task, int stage) {
        if (task < n_tasks) {
            const int seq = task / heads;
            const int h = task - seq * heads;
            const __nv_bfloat16* src = qkv + static_cast<long long>(seq) * T * ld + h * dk;
            const __nv_bfloat16* gsrc = dctx + static_cast<long long>(seq) * T * ld_dctx + h * dk;
            if constexpr (FAST) {
                const uint32_t t0s = wbase_s + 2 * stage * 4 * TILE;
                tile_load_map(t0s, src, lmap, piece);
                tile_load_map(t0s + 2 * TILE, src + sec, lmap, piece);
                tile_load_map(t0s + 4 * TILE, src + 2 * sec, lmap, piece);
                tile_load_map(t0s + 6 * TILE, gsrc, gmap, piece);
            } else {
                __nv_bfloat16* t0 = wbase + stage * 4 * TILE;
                tile_load(t0, src, ld, T, dk, piece, ctid, cnt, PT);
                tile_load(t0 + TILE, src + sec, ld, T, dk, piece, ctid, cnt, PT);
                tile_load(t0 + 2 * TILE, src + 2 * sec, ld, T, dk, piece, ctid, cnt, PT);
                tile_load(t0 + 3 * TILE, gsrc, ld_dctx, T, dk, piece, ctid, cnt, PT);
            }
        }
        cp_commit();
    };
#pragma unroll
    for (int s0 = 0; s0 < kStages - 1; ++s0) prefetch(gw + s0 * W, s0);

    int stage = 0;
    for (int task = gw; task < n_tasks; task += W) {
        cp_wait<kStages - 2>();
        phase_sync();
        // the stage consumed in the previous iteration is free again: refill it before computing this task
        prefetch(task + (kStages - 1) * W, (stage + kStages - 1) % kStages);
        const long long seq = task / heads;
        const int h = task - static_cast<int>(seq) * heads;
        const __nv_bfloat16* q = wbase + stage * 4 * TILE;
        __nv_bfloat16* k = wbase + stage * 4 * TILE + TILE;
        __nv_bfloat16* v = k + TILE;
        const __nv_bfloat16* gg = v + TILE;
        __nv_bfloat16* gout = dqkv + seq * T * static_cast<long long>(ld_d);
        // ---- phase A (row blocks i): P, dS -> smem (bf16); dQ straight to global ----
        // The K / V fragments do not depend on the row block: with two row blocks per task (T <= 32) they are loaded
        // once and kept in registers (the kernel is bound by the shared-memory instruction queue, ncu: stall_mio).
        constexpr bool HOIST = (MT == 2) && !COOP;
        uint32_t hk[HOIST ? KS16 : 1][HOIST ? NTJ : 1][2], hv[HOIST ? KS16 : 1][HOIST ? NTJ : 1][2];
        uint32_t hk8[HOIST && K8T ? NTJ : 1][1], hv8[HOIST && K8T ? NTJ : 1][1];
        if constexpr (HOIST) {
#pragma unroll
            for (int ks = 0; ks < KS16; ++ks)
#pragma unroll
                for (int nt = 0; nt < NTJ; ++nt) {
                    if (nt >= ntj) break;
                    load_b(hk[ks][nt], k, PT, nt * 8, ks * 16, lane);
                    load_b(hv[ks][nt], v, PT, nt * 8, ks * 16, lane);
                }
            if constexpr (K8T) {
#pragma unroll
                for (int nt = 0; nt < NTJ; ++nt) {
                    if (nt >= ntj) break;
                    load_b8(hk8[nt], k, PT, nt * 8, KS16 * 16, lane);
                    load_b8(hv8[nt], v, PT, nt * 8, KS16 * 16, lane);
                }
            }
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
            if (mt * 16 >= T) continue;
            if (COOP && mt != warp) continue;
            float dq[NTD][4];
#pragma unroll
            for (int nd = 0; nd < NTD; ++nd) dq[nd][0] = dq[nd][1] = dq[nd][2] = dq[nd][3] = 0.f;
            float s[NTJ][4], dp[NTJ][4];
#pragma unroll
            for (int nt = 0; nt < NTJ; ++nt) {
                s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
                dp[nt][0] = dp[nt][1] = dp[nt][2] = dp[nt][3] = 0.f;
            }
#pragma unroll
            for (int ks = 0; ks < KS16; ++ks) {
                uint32_t aq[4], ag[4];
                load_a(aq, q, PT, mt * 16, ks * 16, lane);
                load_a(ag, gg, PT, mt * 16, ks * 16, lane);
#pragma unroll
                for (int nt = 0; nt < NTJ; ++nt) {
                    if (nt >= ntj) break;
                    if constexpr (HOIST) {
                        mma_bf16(s[nt], aq, hk[ks][nt]);    // S  = Q K^T
                        mma_bf16(dp[nt], ag, hv[ks][nt]);   // dA = dCtx V^T
                    } else {
                        uint32_t bk[2], bv[2];
                        load_b(bk, k, PT, nt * 8, ks * 16, lane);
                        load_b(bv, v, PT, nt * 8, ks * 16, lane);
                        mma_bf16(s[nt], aq, bk);
                        mma_bf16(dp[nt], ag, bv);
                    }
                }
            }
            if constexpr (K8T) {
                uint32_t aq[2], ag[2];
                load_a8(aq, q, PT, mt * 16, KS16 * 16, lane);
                load_a8(ag, gg, PT, mt * 16, KS16 * 16, lane);
#pragma unroll
                for (int nt = 0; nt < NTJ; ++nt) {
                    if (nt >= ntj) break;
                    if constexpr (HOIST) {
                        mma_bf16_k8(s[nt], aq, hk8[nt]);
                        mma_bf16_k8(dp[nt], ag, hv8[nt]);
                    } else {
                        uint32_t bk[1], bv[1];
                        load_b8(bk, k, PT, nt * 8, KS16 * 16, lane);
                        load_b8(bv, v, PT, nt * 8, KS16 * 16, lane);
                        mma_bf16_k8(s[nt], aq, bk);
                        mma_bf16_k8(dp[nt], ag, bv);
                    }
                }
            }
            const bool dead1 = FIXED && mt * 16 + 8 >= CT;  // rows g+8 of this block are all >= T (folds after unrolling)
            softmax_rows<NTJ>(s, T, t4, ntj, sc, dead1);
            float del0 = 0.f, del1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < NTJ; ++nt) {
                if (nt >= ntj) break;
                del0 += s[nt][0] * dp[nt][0] + s[nt][1] * dp[nt][1];
                if (!dead1) del1 += s[nt][2] * dp[nt][2] + s[nt][3] * dp[nt][3];
            }
            del0 = quad_sum(del0);
            if (!dead1) del1 = quad_sum(del1);
            const bool r0ok = mt * 16 + g < T, r1ok = !dead1 && mt * 16 + g + 8 < T;
#pragma unroll
            for (int nt = 0; nt < NTJ; ++nt) {
                if (nt >= ntj) {  // dead key columns: never stored (the scratch stays zero there), zero dS fragments for dQ
                    dp[nt][0] = dp[nt][1] = dp[nt][2] = dp[nt][3] = 0.f;
                    continue;
                }
                // rows >= T carry garbage (zero Q rows give a uniform softmax): force them to zero, they are
                // k-indices of the phase-B products
                const float p0 = r0ok ? s[nt][0] : 0.f, p1 = r0ok ? s[nt][1] : 0.f;
                const float p2 = r1ok ? s[nt][2] : 0.f, p3 = r1ok ? s[nt][3] : 0.f;
                dp[nt][0] = p0 * (dp[nt][0] - del0) * rs;
                dp[nt][1] = p1 * (dp[nt][1] - del0) * rs;
                dp[nt][2] = p2 * (dp[nt][2] - del1) * rs;
                dp[nt][3] = p3 * (dp[nt][3] - del1) * rs;
                const int col = nt * 8 + 2 * t4;
                *reinterpret_cast<uint32_t*>(ps + (mt * 16 + g) * SP + col) = pack_bf16x2(p0, p1);
                *reinterpret_cast<uint32_t*>(ds + (mt * 16 + g) * SP + col) = pack_bf16x2(dp[nt][0], dp[nt][1]);
                if (!dead1) {  // dead rows are never written by any task of this kernel: they keep their initial zeros
                    *reinterpret_cast<uint32_t*>(ps + (mt * 16 + g + 8) * SP + col) = pack_bf16x2(p2, p3);
                    *reinterpret_cast<uint32_t*>(ds + (mt * 16 + g + 8) * SP + col) = pack_bf16x2(dp[nt][2], dp[nt][3]);
                }
            }
            // dQ = dS K   (A = dS fragments straight from registers, B[k=j][n=d] = K[j][d])
#pragma unroll
            for (int kj = 0; kj < MT; ++kj) {
                if (kj * 16 >= T) break;
                uint32_t a[4];
                a[0] = pack_bf16x2(dp[2 * kj][0], dp[2 * kj][1]);
                a[1] = pack_bf16x2(dp[2 * kj][2], dp[2 * kj][3]);
                a[2] = pack_bf16x2(dp[2 * kj + 1][0], dp[2 * kj + 1][1]);
                a[3] = pack_bf16x2(dp[2 * kj + 1][2], dp[2 * kj + 1][3]);
#pragma unroll
                for (int nd = 0; nd < NTD; ++nd) {
                    uint32_t b[2];
                    load_b_t(b, k, PT, kj * 16, nd * 8, lane);
                    mma_bf16(dq[nd], a, b);
                }
            }
#pragma unroll
            for (int nd = 0; nd < NTD; ++nd) {
                const int col = nd * 8 + 2 * t4;
                if (col >= dk) continue;
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    if (FIXED && mt * 16 + hf * 8 >= CT) continue;  // whole half-block past T: folds after unrolling
                    const int r = mt * 16 + g + hf * 8;
                    if (r >= T) continue;
                    __nv_bfloat16* o = gout + static_cast<size_t>(r) * ld_d + h * dk + col;
                    if (col + 1 < dk && piece >= 4) {
                        *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(dq[nd][2 * hf], dq[nd][2 * hf + 1]);
                    } else {
                        o[0] = __float2bfloat16_rn(dq[nd][2 * hf]);
                        if (col + 1 < dk) o[1] = __float2bfloat16_rn(dq[nd][2 * hf + 1]);
                    }
                }
            }
        }
        phase_sync();
        // ---- phase B (row blocks j): dK = dS^T Q, dV = P^T dCtx ----
        // (K and V tiles are dead after phase A: each row block's result goes straight into them)
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
            if (mt * 16 >= T) continue;
            if (COOP && mt != warp) continue;
            float dkk[NTD][4], dvv[NTD][4];
#pragma unroll
            for (int nd = 0; nd < NTD; ++nd) {
                dkk[nd][0] = dkk[nd][1] = dkk[nd][2] = dkk[nd][3] = 0.f;
                dvv[nd][0] = dvv[nd][1] = dvv[nd][2] = dvv[nd][3] = 0.f;
            }
#pragma unroll
            for (int ki = 0; ki < MT; ++ki) {
                if (ki * 16 >= T) break;
                uint32_t ad[4], ap[4];
                load_a_t(ad, ds, SP, mt * 16, ki * 16, lane);
                load_a_t(ap, ps, SP, mt * 16, ki * 16, lane);
#pragma unroll
                for (int nd = 0; nd < NTD; ++nd) {
                    uint32_t bq[2], bg[2];
                    load_b_t(bq, q, PT, ki * 16, nd * 8, lane);
                    load_b_t(bg, gg, PT, ki * 16, nd * 8, lane);
                    mma_bf16(dkk[nd], ad, bq);
                    mma_bf16(dvv[nd], ap, bg);
                }
            }
#pragma unroll
            for (int nd = 0; nd < NTD; ++nd) {
                const int col = nd * 8 + 2 * t4;
                if (col >= dk) continue;
                const bool pair = col + 1 < dk;  // odd d_k: keep the zero padding column intact
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    if (FIXED && mt * 16 + hf * 8 >= CT) continue;  // whole half-block past T: folds after unrolling
                    const int r = mt * 16 + g + hf * 8;
                    if (r >= T) continue;
                    *reinterpret_cast<uint32_t*>(k + r * PT + col) = pack_bf16x2(dkk[nd][2 * hf], pair ? dkk[nd][2 * hf + 1] : 0.f);
                    *reinterpret_cast<uint32_t*>(v + r * PT + col) = pack_bf16x2(dvv[nd][2 * hf], pair ? dvv[nd][2 * hf + 1] : 0.f);
                }
            }
        }
        phase_sync();
        if constexpr (FAST) {
            tile_store_map(k, gout + sec + h * dk, smap, piece);
            tile_store_map(v, gout + 2 * sec + h * dk, smap, piece);
        } else {
            tile_store(k, gout + sec + h * dk, ld_d, T, dk, piece, ctid, cnt, PT);
            tile_store(v, gout + 2 * sec + h * dk, ld_d, T, dk, piece, ctid, cnt, PT);
        }
        if (h == 0 && sec > d) {  // section padding of dQ | dK | dV: zeros (it is a contraction index of the projection backward)
            const int pw = sec - d;
            for (int i = ctid; i < T * 3 * pw; i += cnt) {
                const int r = i / (3 * pw), rem = i - r * 3 * pw, sct = rem / pw;
                gout[static_cast<size_t>(r) * ld_d + sct * sec + d + (rem - sct * pw)] = __float2bfloat16_rn(0.f);
            }
        }
        phase_sync();
        stage = (stage + 1) % kStages;
    }
    cp_wait<0>();
}

template <int NTD, bool FAST, bool FIXED, bool COOP>
int launch_mma(bool bwd, const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int T, int heads, int dk,
               void* out, int ld_out, const Dropout& drop, cudaStream_t stream) {
    const long long tasks = n_seq * heads;
    NR_REQUIRE(tasks < (1ll << 31), "mhsa: too many (sequence, head) tasks");
    constexpr int TP = tile_rows(COOP);
    constexpr int PT = FIXED ? kPitch24 : kPitch;
    const size_t tile = sizeof(__nv_bfloat16) * T * PT;
    const int sets = COOP ? 1 : kWarps;  // tile sets per CTA: one per warp, or one shared by the cooperative CTA
    const size_t smem_f = sets * kStages * 3 * tile + sizeof(__nv_bfloat16) * (TP - T) * PT;
    const size_t smem_b = sets * (kStages * 4 * tile + sizeof(__nv_bfloat16) * 2 * TP * (TP + 8));
    const size_t smem = bwd ? smem_b : smem_f;
    NR_REQUIRE(smem <= 227 * 1024, "mhsa: tile set of %zu bytes exceeds shared memory", smem);
    const int per_sm = std::max<int>(1, std::min<size_t>(COOP ? 3 : (bwd ? 6 : 8), (224 * 1024) / (smem + 1024)));
    const int grid = static_cast<int>(std::min<long long>(ceil_div(static_cast<int>(std::min<long long>(tasks, 1 << 30)), COOP ? 1 : kWarps),
                                                          static_cast<long long>(num_sms()) * per_sm));
    if (!bwd) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(mhsa_mma_fwd_kernel<NTD, FAST, FIXED, COOP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        mhsa_mma_fwd_kernel<NTD, FAST, FIXED, COOP><<<grid, kWarps * 32, smem, stream>>>(static_cast<const __nv_bfloat16*>(qkv), ld_qkv, sec, n_seq, T,
                                                                                       heads, dk, static_cast<__nv_bfloat16*>(out), ld_out, drop);
    } else {
        NR_CHECK_CUDA(cudaFuncSetAttribute(mhsa_mma_bwd_kernel<NTD, FAST, FIXED, COOP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        mhsa_mma_bwd_kernel<NTD, FAST, FIXED, COOP><<<grid, kWarps * 32, smem, stream>>>(static_cast<const __nv_bfloat16*>(qkv), ld_qkv, sec,
                                                                                       static_cast<const __nv_bfloat16*>(dctx), ld_dctx, n_seq, T,
                                                                                       heads, dk, static_cast<__nv_bfloat16*>(out), ld_out);
    }
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <bool FAST, bool COOP>
int launch_dk(bool bwd, const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int T, int heads, int dk,
              void* out, int ld_out, const Dropout& drop, cudaStream_t stream) {
    if (dk <= 16) return launch_mma<2, FAST, false, COOP>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
    if (dk <= 24) return launch_mma<3, FAST, false, COOP>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
    return launch_mma<4, FAST, false, COOP>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
}

// Picks the kernel from the input.  T > 32 runs on cooperative CTAs (one task per CTA), T <= 32 on per-warp tasks.  Both take
// the fixed-shape kernel for the reference's head shape when its rows move in 8-byte pieces.  Otherwise the per-warp tasks use
// the per-lane copy plan when it covers the tile (up to kMaxP * 32 pieces of >= 4 bytes) and the copy loops when it does not.
int dispatch(bool bwd, const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int T, int heads, int dk,
             void* out, int ld_out, const Dropout& drop, cudaStream_t stream) {
    const bool coop = T > 32;
    const int piece = bwd ? piece_bytes_bwd(dk, ld_qkv, ld_dctx, sec, ld_out) : piece_bytes(dk, ld_qkv, ld_out, sec);
    if (piece == 8 && T == fixed_T(coop) && dk == kFixedDk && heads == kFixedHeads) {  // d_k 20: the NTD 3 class
        if (coop) return launch_mma<3, false, true, true>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
        // per-warp: the copy plan always covers it (20 rows x 5 pieces of 8 bytes)
        return launch_mma<3, true, true, false>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
    }
    if (coop) return launch_dk<false, true>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
    const bool fast = piece >= 4 && T * (dk / (piece / 2)) <= kMaxP * 32;
    if (fast) return launch_dk<true, false>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
    return launch_dk<false, false>(bwd, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, out, ld_out, drop, stream);
}

// The shape contract both directions share (include/newsrec_b200.h), checked before anything is launched.  Every pitch is a
// multiple of 8, which the context dropout's mask needs (Dropout in nr_common.cuh: a pitch that is a multiple of 4).
int check_core_shape(long long n_seq, int T, int heads, int dk, int sec, int ld_qkv) {
    NR_REQUIRE(n_seq >= 0, "mhsa: n_seq=%lld is negative", n_seq);
    NR_REQUIRE(heads >= 1, "mhsa: heads=%d, need at least one head", heads);
    NR_REQUIRE(T >= 1 && T <= 64, "mhsa: sequence length %d not in [1,64]", T);
    NR_REQUIRE(dk >= 2 && dk <= 32, "mhsa: head size d_k=%d not in [2,32]", dk);
    NR_REQUIRE(sec >= static_cast<long long>(heads) * dk && ld_qkv >= 3ll * sec, "mhsa: Q|K|V section stride %d / pitch %d too small for d=%lld",
               sec, ld_qkv, static_cast<long long>(heads) * dk);
    NR_REQUIRE(ld_qkv % 8 == 0, "mhsa: Q|K|V pitch %d is not a multiple of 8", ld_qkv);
    return 0;
}

}  // namespace

int mhsa_core_fwd(const void* qkv, int ld_qkv, int sec, long long n_seq, int T, int heads, int dk, void* ctx, int ld_ctx, DropoutCfg drop,
                  cudaStream_t stream) {
    NR_PROPAGATE(check_core_shape(n_seq, T, heads, dk, sec, ld_qkv));
    NR_REQUIRE(ld_ctx >= heads * dk + 1, "mhsa: context pitch %d has no room for the ones column", ld_ctx);
    NR_REQUIRE(ld_ctx % 8 == 0, "mhsa: context pitch %d is not a multiple of 8", ld_ctx);
    NR_REQUIRE(drop.p >= 0.f && drop.p < 1.f, "mhsa: dropout p=%f not in [0, 1)", drop.p);
    if (n_seq == 0) return 0;
    ProfScope ps("mhsa_core_fwd", static_cast<int>(n_seq), T, heads * dk, stream);
    if (mhsa_title_fwd_supported(T, dk, heads, sec, ld_qkv, ld_ctx))  // the news encoder's shape: whole titles per CTA, TMA in / out
        return mhsa_title_fwd(qkv, ld_qkv, sec, n_seq, heads, ctx, ld_ctx, drop, stream);
    return dispatch(false, qkv, ld_qkv, sec, nullptr, 0, n_seq, T, heads, dk, ctx, ld_ctx, Dropout::make(drop.p, drop.seed), stream);
}

int mhsa_core_bwd(const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int T, int heads, int dk,
                  void* dqkv, int ld_dqkv, cudaStream_t stream, const PaddingTitles* pad) {
    NR_PROPAGATE(check_core_shape(n_seq, T, heads, dk, sec, ld_qkv));
    NR_REQUIRE(ld_dqkv >= 3 * sec && ld_dctx >= heads * dk, "mhsa: dQ|dK|dV pitch %d / context-gradient pitch %d too small for sec=%d d=%d",
               ld_dqkv, ld_dctx, sec, heads * dk);
    NR_REQUIRE(ld_dctx % 8 == 0 && ld_dqkv % 8 == 0, "mhsa: context-gradient pitch %d / dQ|dK|dV pitch %d is not a multiple of 8", ld_dctx,
               ld_dqkv);
    if (n_seq == 0) return 0;
    ProfScope ps("mhsa_core_bwd", static_cast<int>(n_seq), T, heads * dk, stream);
    if (mhsa_title_bwd_supported(T, dk, heads, sec, ld_qkv, ld_dctx, ld_dqkv))  // the news encoder's shape: whole titles per CTA, TMA in / out
        return mhsa_title_bwd(qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, heads, dqkv, ld_dqkv, stream, pad);
    NR_REQUIRE(pad == nullptr, "mhsa: padding titles need the title-level kernel");
    return dispatch(true, qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, dqkv, ld_dqkv, Dropout::make(0.f, 0), stream);
}

}  // namespace nr
