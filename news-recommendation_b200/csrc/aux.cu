// Memory-bound companions of the wgmma GEMMs: the fp32 -> bf16 row conversions, the embedding-row gather, pooling-backward
// row dots, the dot-product click scorer, the fp32 attention of the precise user encoder, impression scoring, metrics, ranks
// and the prediction text, the batch feed.  All HBM-bound integer/byte or small-reduction work: coalesced 16-byte accesses,
// warp-shuffle reductions, no tensor cores.
#include <algorithm>

#include <cub/device/device_scan.cuh>

#include "nr_common.cuh"
#include "nr_ops.h"

namespace nr {

// ------------------------------------------------------------------------------------------------
// fp32 rows -> zero-padded bf16 planes (Bf16Rows, nr_ops.h)
// ------------------------------------------------------------------------------------------------
// One thread per 16-byte chunk (8 columns), grid-stride over the rows x chunks of a job: x is formed once per element and every
// requested plane is written from it.  Chunks are taken row by row, so neighbouring threads read neighbouring columns; for strided
// columns (a transpose) they are taken column by column instead, so that neighbouring threads read neighbouring rows and the
// loads coalesce.  Several jobs share one launch (blockIdx.y = job): the packed and transposed weights of an encoder are a few
// hundred rows each, and as separate launches they cost more in launch gaps than in work.  A single job runs in 512-thread
// blocks with its descriptor at fixed parameter offsets; a batch runs in 128-thread blocks, so that its small jobs spread over
// more SMs.
template <int N>
struct Bf16Jobs {
    Bf16Rows job[N];
};
__device__ __forceinline__ uint4 pack_bf16x8(const float (&v)[8]) {
    return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}
template <int N, int kThreads>
__global__ void __launch_bounds__(kThreads) rows_to_bf16_kernel(const __grid_constant__ Bf16Jobs<N> jobs) {
    const Bf16Rows& j = jobs.job[N == 1 ? 0 : blockIdx.y];
    const int D = j.D, T = j.T, chunks = j.width >> 3, n_rows = static_cast<int>(j.n_rows);  // n_rows * chunks < 2^30
    const bool by_col = j.s_col != 1;
    __nv_bfloat16* const hi = static_cast<__nv_bfloat16*>(j.hi);
    __nv_bfloat16* const lo = static_cast<__nv_bfloat16*>(j.lo);
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n_rows * chunks; i += gridDim.x * kThreads) {
        const int c = by_col ? i / n_rows : i % chunks;
        const int r = by_col ? i - c * n_rows : i / chunks;
        const int col = c * 8;
        const int seq = T == 1 ? r : r / T;
        const int tok = r - seq * T;
        const float* sp = j.src + seq * j.s_seq + tok * j.s_tok;
        float x[8];
        if (j.s_col == 1 && col + 8 <= D && (reinterpret_cast<uintptr_t>(sp + col) & 15) == 0) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(sp + col)), b = __ldg(reinterpret_cast<const float4*>(sp + col) + 1);
            x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] = col + e < D ? __ldg(sp + (col + e) * j.s_col) : 0.f;
        }
        if (j.pos != nullptr) {
            const float* pp = j.pos + tok * D;
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (col + e < D) x[e] += __ldg(pp + col + e);
        }
        if (hi != nullptr) {
            float h[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) h[e] = j.ones_col && col + e == D ? 1.0f : x[e];
            *reinterpret_cast<uint4*>(hi + static_cast<long long>(r) * j.ld_hi + col) = pack_bf16x8(h);
        }
        if (lo != nullptr) {
            float l[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) l[e] = x[e] - bf16_round(x[e]);
            *reinterpret_cast<uint4*>(lo + static_cast<long long>(r) * j.ld_lo + col) = pack_bf16x8(l);
        }
    }
}
static bool plane_ok(const void* p, int ld, int width) {
    return p == nullptr || ((reinterpret_cast<uintptr_t>(p) & 15) == 0 && ld % 8 == 0 && ld >= width);
}
int rows_to_bf16(const Bf16Rows* jobs, int n_jobs, Bf16Op op, cudaStream_t stream) {
    NR_REQUIRE(n_jobs >= 0 && n_jobs <= kBf16RowsJobs, "%s: %d jobs (at most %d per launch)", op.name, n_jobs, kBf16RowsJobs);
    Bf16Jobs<kBf16RowsJobs> a;
    int n = 0;
    long long chunks = 0, biggest = 0;  // of the largest job
    for (int i = 0; i < n_jobs; ++i) {
        const Bf16Rows& j = jobs[i];
        NR_REQUIRE(j.src && (j.hi || j.lo) && j.n_rows >= 0 && j.T >= 1 && j.D >= 0 && j.width % 8 == 0 &&
                       j.width >= j.D + (j.hi && j.ones_col ? 1 : 0) && plane_ok(j.hi, j.ld_hi, j.width) && plane_ok(j.lo, j.ld_lo, j.width),
                   "%s: job %d: n_rows=%lld T=%d D=%d width=%d ld_hi=%d ld_lo=%d (null or misaligned operand?)", op.name, i, j.n_rows, j.T,
                   j.D, j.width, j.ld_hi, j.ld_lo);
        NR_REQUIRE(j.n_rows * (j.width / 8) < (1ll << 30), "%s: job %d: %lld rows of %d columns", op.name, i, j.n_rows, j.width);
        if (j.n_rows == 0 || j.width == 0) continue;
        chunks = std::max(chunks, j.n_rows * (j.width / 8));
        biggest = std::max(biggest, j.n_rows * j.width);
        a.job[n++] = j;
    }
    if (n == 0) return 0;
    // one job: its shape; a batch: the job count and the largest job's elements
    ProfScope ps(op.name, n_jobs == 1 ? static_cast<int>(a.job[0].n_rows) : n_jobs,
                 n_jobs == 1 ? a.job[0].D : static_cast<int>(std::min<long long>(biggest, 1 << 30)), n_jobs == 1 ? a.job[0].width : 0,
                 stream);
    const int threads = n == 1 ? 512 : 128;
    const dim3 grid(static_cast<unsigned>(std::min<long long>((chunks + threads - 1) / threads, 148ll * op.blocks_per_sm)),
                    static_cast<unsigned>(n));
    if (n == 1) rows_to_bf16_kernel<1, 512><<<grid, 512, 0, stream>>>(Bf16Jobs<1>{a.job[0]});
    else rows_to_bf16_kernel<kBf16RowsJobs, 128><<<grid, 128, 0, stream>>>(a);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Embedding-row gather: one warp per token, 16-byte lanes.  The copy is bit exact (bf16 table rows).
// Column D of every gathered row is set to 1.0 (bias-gradient trick), columns after it stay 0.
// ------------------------------------------------------------------------------------------------
// one thread = one 16-byte chunk COLUMN: a block covers kGatherThreads / chunks consecutive token rows per iteration
// (consecutive threads copy consecutive chunks: coalesced), so the chunk index and the row slot are computed once and
// the loop carries no division (the flat-index version spent most of its instructions on 64-bit div/mod);
// dropout draws ONE counter hash per 4 aligned columns (two per chunk)
constexpr int kGatherThreads = 320;
__global__ void __launch_bounds__(kGatherThreads) gather_rows_kernel(const long long* __restrict__ ids, long long n_tok, int T,
                                                                   const uint4* __restrict__ table, int V, int D, int ld,
                                                                   uint4* __restrict__ X, int ld_x, int padded, Dropout drop,
                                                                   int* bad_flag, const int* __restrict__ index,
                                                                   const int* __restrict__ n_live) {
    const int chunks = ld >> 3;  // 16-byte chunks per table row
    const int x_chunks = ld_x >> 3;
    const int rows_per_it = kGatherThreads / chunks;
    const int rl = threadIdx.x / chunks, c = threadIdx.x - rl * chunks;
    if (rl >= rows_per_it) return;
    const long long stride = static_cast<long long>(gridDim.x) * rows_per_it;
    // compact rows (index non-null): X row i < M' is token index[i]; the rows [M', round_up(M', 64)) below n_tok are zero rows
    long long n_rows = n_tok;
    if (index != nullptr) {
        n_rows = __ldg(n_live);
        const long long tail_end = min(n_tok, (n_rows + 63) / 64 * 64);
        for (long long r = static_cast<long long>(blockIdx.x) * rows_per_it + rl + n_rows; r < tail_end; r += stride)
            X[r * x_chunks + c] = make_uint4(0, 0, 0, 0);
    }
    const auto token = [&](long long i) -> long long { return index != nullptr ? __ldg(index + i) : i; };
    long long i = static_cast<long long>(blockIdx.x) * rows_per_it + rl;
    // software pipeline: the (id -> table row) loads of the NEXT row are in flight while this one is stored
    long long tok = i < n_rows ? token(i) : 0;
    long long n_id = i < n_rows ? __ldg(ids + tok) : 0;
    if (i < n_rows && (n_id < 0 || n_id >= V)) { atomicExch(bad_flag, 1); n_id = 0; }
    uint4 n_u = i < n_rows ? __ldg(table + n_id * chunks + c) : make_uint4(0, 0, 0, 0);
    const int col = c * 8;
    for (; i < n_rows; i += stride) {
        uint4 u = n_u;
        const long long cur = tok, i2 = i + stride;
        if (i2 < n_rows) {
            tok = token(i2);
            n_id = __ldg(ids + tok);
            if (n_id < 0 || n_id >= V) { atomicExch(bad_flag, 1); n_id = 0; }
            n_u = __ldg(table + n_id * chunks + c);
        }
        long long xr = cur;  // the row of the token: it keys the dropout draw
        int t = 0;
        if (padded) {
            const long long seg = cur / T;
            t = static_cast<int>(cur - seg * T);
            xr = seg * (T + 2) + 1 + t;
        }
        uint32_t w[4] = {u.x, u.y, u.z, u.w};
        if (drop.active()) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float m[4];
                drop.mask4_group(static_cast<uint64_t>(xr) * (ld_x >> 2) + (col >> 2) + h, m);  // ld_x % 8 == 0
                const float2 f0 = unpack_bf16x2(w[2 * h]), f1 = unpack_bf16x2(w[2 * h + 1]);
                w[2 * h] = pack_bf16x2(f0.x * m[0], f0.y * m[1]);
                w[2 * h + 1] = pack_bf16x2(f1.x * m[2], f1.y * m[3]);
            }
        }
        if (D >= col && D < col + 8) {  // ones column, zeros behind it
            __nv_bfloat16* e = reinterpret_cast<__nv_bfloat16*>(w);
            for (int j = D - col; j < 8; ++j) e[j] = __float2bfloat16_rn(j == D - col ? 1.0f : 0.f);
        }
        X[(index != nullptr ? i : xr) * x_chunks + c] = make_uint4(w[0], w[1], w[2], w[3]);
        if (padded) {
            if (t == 0) X[(xr - 1) * x_chunks + c] = make_uint4(0, 0, 0, 0);
            if (t == T - 1) X[(xr + 1) * x_chunks + c] = make_uint4(0, 0, 0, 0);
        }
    }
}
int gather_rows(const long long* ids, long long n_tok, int T, const void* table, int V, int D, int ld_table, void* X,
                int ld_x, int padded, DropoutCfg drop, int* bad_id_flag, cudaStream_t stream, const LiveTokens* live) {
    if (n_tok == 0) return 0;
    NR_REQUIRE(ld_table % 8 == 0 && ld_x % 8 == 0 && ld_x >= ld_table && ld_table >= D + 1 && ld_table / 8 <= kGatherThreads,
               "gather_rows: pitch %d/%d for D=%d", ld_table, ld_x, D);
    NR_REQUIRE(live == nullptr || (!padded && ld_x == ld_table && live->index && live->offset),
               "gather_rows: compact rows need the unpadded layout, ld_x == ld_table and the live tokens' index");
    const int rows_per_it = kGatherThreads / (ld_table / 8);
    const int blocks = static_cast<int>(std::min<long long>((n_tok + rows_per_it - 1) / rows_per_it, 148 * 6));
    ProfScope ps("gather_rows", static_cast<int>(n_tok), D, ld_x, stream);
    gather_rows_kernel<<<blocks, kGatherThreads, 0, stream>>>(ids, n_tok, T, static_cast<const uint4*>(table), V, D, ld_table,
                                                   static_cast<uint4*>(X), ld_x, padded, Dropout::make(drop.p, drop.seed),
                                                   bad_id_flag, live != nullptr ? live->index : nullptr,
                                                   live != nullptr ? live->offset + n_tok / T : nullptr);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// pooling backward, scalar part: dw_r = dOut[seg] . X_r ; dscore_r = w_r (dw_r - sum_seg w dw)
// ------------------------------------------------------------------------------------------------
// Two phases inside one block (= a few segments): (1) every warp takes rows round-robin and keeps the 16-byte loads of
// up to 4 rows in flight before reducing (the first version walked rows one by one and was latency bound at ~1.3 TB/s);
// (2) one thread per row turns the row dots into dscore.
constexpr int kDsSegs = 6;    // segments per block iteration
__global__ void __launch_bounds__(256) pool_dscore_kernel(const __nv_bfloat16* __restrict__ X, int lda, int D,
                                                          long long n_seg, int seg_len, const float* __restrict__ w,
                                                          const float* __restrict__ dout, int ldo,
                                                          float* __restrict__ dscore) {
    extern __shared__ float s_dw[];  // [kDsSegs * seg_len]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = D >> 3;
    const long long n_groups = (n_seg + kDsSegs - 1) / kDsSegs;
    for (long long grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
        const long long seg0 = grp * kDsSegs;
        const int nsg = static_cast<int>(min(static_cast<long long>(kDsSegs), n_seg - seg0));
        const int nrows = nsg * seg_len;
        for (int r0 = warp * 4; r0 < nrows; r0 += 8 * 4) {
            uint4 u[4][2];
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int r = r0 + k;
                const uint4* xr = reinterpret_cast<const uint4*>(X + (seg0 * seg_len + r) * static_cast<long long>(lda));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int c = lane + 32 * h;
                    u[k][h] = (r < nrows && c < chunks) ? __ldg(xr + c) : make_uint4(0, 0, 0, 0);
                }
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int r = r0 + k;
                if (r >= nrows) break;
                const float* dob = dout + (seg0 + r / seg_len) * ldo;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int c = lane + 32 * h;
                    if (c < chunks) {
                        const float4 d0 = *reinterpret_cast<const float4*>(dob + c * 8);
                        const float4 d1 = *reinterpret_cast<const float4*>(dob + c * 8 + 4);
                        const uint4 v = u[k][h];
                        const float2 f0 = unpack_bf16x2(v.x), f1 = unpack_bf16x2(v.y), f2 = unpack_bf16x2(v.z), f3 = unpack_bf16x2(v.w);
                        float a = acc[k];
                        a = fmaf(f0.x, d0.x, a); a = fmaf(f0.y, d0.y, a); a = fmaf(f1.x, d0.z, a); a = fmaf(f1.y, d0.w, a);
                        a = fmaf(f2.x, d1.x, a); a = fmaf(f2.y, d1.y, a); a = fmaf(f3.x, d1.z, a); a = fmaf(f3.y, d1.w, a);
                        acc[k] = a;
                    }
                }
                // columns beyond 64 chunks (D > 512) and the D % 8 tail
                const __nv_bfloat16* xe = X + (seg0 * seg_len + r) * static_cast<long long>(lda);
                for (int c = 64 + lane; c < chunks; c += 32) {
                    const uint4 v = __ldg(reinterpret_cast<const uint4*>(xe) + c);
                    const uint32_t vw[4] = {v.x, v.y, v.z, v.w};
                    for (int j = 0; j < 4; ++j) {
                        const float2 f = unpack_bf16x2(vw[j]);
                        acc[k] = fmaf(f.x, dob[c * 8 + 2 * j], acc[k]);
                        acc[k] = fmaf(f.y, dob[c * 8 + 2 * j + 1], acc[k]);
                    }
                }
                for (int c = chunks * 8 + lane; c < D; c += 32) acc[k] = fmaf(__bfloat162float(xe[c]), dob[c], acc[k]);
                const float tot = warp_sum(acc[k]);
                if (lane == 0) s_dw[r] = tot;
            }
        }
        __syncthreads();
        for (int r = threadIdx.x; r < nrows; r += blockDim.x) {
            const int sgi = r / seg_len;
            const float* wr = w + (seg0 + sgi) * seg_len;
            const float* dwr = s_dw + sgi * seg_len;
            float dot = 0.f;
            for (int t = 0; t < seg_len; ++t) dot = fmaf(wr[t], dwr[t], dot);
            dscore[seg0 * seg_len + r] = wr[r - sgi * seg_len] * (s_dw[r] - dot);
        }
        __syncthreads();
    }
}
// Title-level shape (seg_len <= 32, D <= 512): one WARP per segment, no shared memory and no block barrier.  The
// segment's dOut chunk stays in registers for all its rows, 5 rows x 2 16-byte loads are in flight per lane, and the
// per-row totals come out of one 31-shuffle transpose reduction (lane t ends with dw_t) instead of 5 shuffles per row.
__global__ void __launch_bounds__(256) pool_dscore_warp_kernel(const __nv_bfloat16* __restrict__ X, int lda, int D,
                                                               long long n_seg, int seg_len, const float* __restrict__ w,
                                                               const float* __restrict__ dout, int ldo,
                                                               float* __restrict__ dscore) {
    const int lane = threadIdx.x & 31;
    const int chunks = (D + 7) >> 3;  // the last one may be half valid (D % 8 == 4): its dOut and X halves are zeroed below
    const long long wstride = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
    for (long long seg = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); seg < n_seg; seg += wstride) {
        const float* dob = dout + seg * ldo;
        float4 dd[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = lane + 32 * h;
            dd[h][0] = (c < chunks && c * 8 + 4 <= D) ? *reinterpret_cast<const float4*>(dob + c * 8) : make_float4(0.f, 0.f, 0.f, 0.f);
            dd[h][1] = (c < chunks && c * 8 + 8 <= D) ? *reinterpret_cast<const float4*>(dob + c * 8 + 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const uint4* xs = reinterpret_cast<const uint4*>(X + seg * seg_len * static_cast<long long>(lda));
        const int pitch16 = lda >> 3;
        float pr[32];
#pragma unroll
        for (int tb = 0; tb < 32; tb += 4) {
            uint4 u[4][2];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int t = tb + k;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int c = lane + 32 * h;
                    u[k][h] = (t < seg_len && c < chunks) ? __ldg(xs + static_cast<long long>(t) * pitch16 + c) : make_uint4(0, 0, 0, 0);
                    // the half past D of a half-valid chunk is X's pitch (the ones column, then anything): 0 * NaN would be NaN
                    if (c * 8 + 8 > D) u[k][h].z = u[k][h].w = 0u;
                }
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float a = 0.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint4 v = u[k][h];
                    const float2 f0 = unpack_bf16x2(v.x), f1 = unpack_bf16x2(v.y), f2 = unpack_bf16x2(v.z), f3 = unpack_bf16x2(v.w);
                    a = fmaf(f0.x, dd[h][0].x, a); a = fmaf(f0.y, dd[h][0].y, a); a = fmaf(f1.x, dd[h][0].z, a); a = fmaf(f1.y, dd[h][0].w, a);
                    a = fmaf(f2.x, dd[h][1].x, a); a = fmaf(f2.y, dd[h][1].y, a); a = fmaf(f3.x, dd[h][1].z, a); a = fmaf(f3.y, dd[h][1].w, a);
                }
                pr[tb + k] = a;
            }
            if (tb + 4 >= seg_len) {  // warp-uniform: the remaining row slots stay zero
#pragma unroll
                for (int t = tb + 4; t < 32; ++t) pr[t] = 0.f;
                break;
            }
        }
        const float dw = warp_transpose_sum32(pr);  // lane t: dOut . X_t
        const float wt = lane < seg_len ? __ldg(w + seg * seg_len + lane) : 0.f;
        const float dot = warp_sum(wt * dw);
        if (lane < seg_len) dscore[seg * seg_len + lane] = wt * (dw - dot);
    }
}

int pool_dscore_check(int lda, int D, int seg_len, int ldo) {
    NR_REQUIRE(seg_len >= 1 && seg_len <= 128 && D % 4 == 0 && ldo % 4 == 0 && lda % 8 == 0, "pool_dscore: seg_len=%d D=%d ldo=%d lda=%d",
               seg_len, D, ldo, lda);
    return 0;
}

int pool_dscore(const void* X, int lda, int D, long long n_seg, int seg_len, const float* w, const float* dout, int ldo,
                float* dscore, cudaStream_t stream) {
    if (n_seg == 0) return 0;
    NR_PROPAGATE(pool_dscore_check(lda, D, seg_len, ldo));
    const long long groups = (n_seg + kDsSegs - 1) / kDsSegs;
    const int blocks = static_cast<int>(std::min<long long>(groups, 148 * 8));
    ProfScope ps("pool_dscore", static_cast<int>(n_seg), seg_len, D, stream);
    if (seg_len <= 32 && D <= 512) {
        const int wblocks = static_cast<int>(std::min<long long>((n_seg + 7) / 8, 148 * 8));
        pool_dscore_warp_kernel<<<wblocks, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(X), lda, D, n_seg, seg_len, w, dout, ldo,
                                                             dscore);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    pool_dscore_kernel<<<blocks, 256, sizeof(float) * kDsSegs * seg_len, stream>>>(
        static_cast<const __nv_bfloat16*>(X), lda, D, n_seg, seg_len, w, dout, ldo, dscore);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Extended weight gradient [rows][ld] (columns [0,D) = dW, column D = db from the ones-column trick) -> accumulated
// into the parameters' own .grad storage, and cleared for the next step (the buffer is a persistent workspace).
// Replaces, per weight, ~4 framework kernels (2 slice copies + 2 AccumulateGrad adds + the zero fill).
// ------------------------------------------------------------------------------------------------
__global__ void accumulate_ext_grad_kernel(float* __restrict__ ext, int rows, int ld, int D, float* __restrict__ dW,
                                           float* __restrict__ db) {
    const long long n = static_cast<long long>(rows) * (D + 1);
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int r = static_cast<int>(i / (D + 1)), c = static_cast<int>(i - static_cast<long long>(r) * (D + 1));
        float* src = ext + static_cast<size_t>(r) * ld + c;
        const float v = *src;
        *src = 0.f;
        if (c < D) dW[static_cast<size_t>(r) * D + c] += v;
        else if (db != nullptr) db[r] += v;
    }
}
int accumulate_ext_grad(float* ext, int rows, int ld, int D, float* dW, float* db, cudaStream_t stream) {
    if (rows == 0) return 0;
    NR_REQUIRE(ld >= D + 1, "accumulate_ext_grad: pitch %d < D+1 = %d", ld, D + 1);
    const long long n = static_cast<long long>(rows) * (D + 1);
    const int blocks = static_cast<int>(std::min<long long>((n + 255) / 256, 148 * 8));
    accumulate_ext_grad_kernel<<<blocks, 256, 0, stream>>>(ext, rows, ld, D, dW, db);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// ReLU backward + cast:  dst = dy * (relu_out > 0)  -> zero padded bf16 rows
// ------------------------------------------------------------------------------------------------
__global__ void relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ ro, long long n, int N, int ld_dy,
                                __nv_bfloat16* __restrict__ dst, int ldn) {
    const long long total = n * ldn;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long r = i / ldn;
        const int c = static_cast<int>(i - r * ldn);
        float v = 0.f;
        if (c < N) {
            v = dy[r * ld_dy + c];
            if (ro != nullptr && !(ro[r * ld_dy + c] > 0.f)) v = 0.f;
        }
        dst[i] = __float2bfloat16_rn(v);
    }
}
int relu_bwd_to_bf16(const float* dy, const float* relu_out, long long n, int N, int ld_dy, void* dst, int ldn, cudaStream_t stream) {
    if (n == 0) return 0;
    ProfScope ps("relu_bwd_to_bf16", static_cast<int>(n), N, ldn, stream);
    const int blocks = static_cast<int>(std::min<long long>((n * ldn + 255) / 256, 148 * 16));
    relu_bwd_kernel<<<blocks, 256, 0, stream>>>(dy, relu_out, n, N, ld_dy, static_cast<__nv_bfloat16*>(dst), ldn);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// fp32 embedding rows (category / user tables): gather forward, red.add scatter backward
// ------------------------------------------------------------------------------------------------
__global__ void emb_f32_fwd_kernel(const long long* __restrict__ ids, long long n, const float* __restrict__ table, int V, int D,
                                   float* __restrict__ out, int* bad_flag) {
    const int lane = threadIdx.x & 31;
    const long long w0 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
    const long long nw = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
    for (long long i = w0; i < n; i += nw) {
        long long id = ids[i];
        if (id < 0 || id >= V) {
            if (lane == 0) atomicExch(bad_flag, 1);
            id = 0;
        }
        for (int c = lane; c < D; c += 32) out[i * D + c] = table[id * D + c];
    }
}
__global__ void emb_f32_bwd_kernel(const long long* __restrict__ ids, long long n, const float* __restrict__ dout, int V, int D,
                                   float* __restrict__ dtable) {
    const int lane = threadIdx.x & 31;
    const long long w0 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
    const long long nw = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
    for (long long i = w0; i < n; i += nw) {
        const long long id = ids[i];
        if (id <= 0 || id >= V) continue;  // padding_idx; out-of-range ids were flagged by the forward lookup
        for (int c = lane; c < D; c += 32) red_add_f32(dtable + id * D + c, dout[i * D + c]);
    }
}
int embedding_f32_fwd(const long long* ids, long long n, const float* table, int V, int D, float* out, int* bad_id_flag,
                      cudaStream_t stream) {
    if (n == 0) return 0;
    ProfScope ps("embedding_f32_fwd", static_cast<int>(n), D, V, stream);
    const int blocks = static_cast<int>(std::min<long long>((n + 7) / 8, 148 * 8));
    emb_f32_fwd_kernel<<<blocks, 256, 0, stream>>>(ids, n, table, V, D, out, bad_id_flag);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}
int embedding_f32_bwd(const long long* ids, long long n, const float* dout, int V, int D, float* dtable, cudaStream_t stream) {
    if (n == 0) return 0;
    ProfScope ps("embedding_f32_bwd", static_cast<int>(n), D, 0, stream);
    const int blocks = static_cast<int>(std::min<long long>((n + 7) / 8, 148 * 8));
    emb_f32_bwd_kernel<<<blocks, 256, 0, stream>>>(ids, n, dout, V, D, dtable);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// dot-product click predictor (reference dot_product.py:8-19): one warp per (impression, candidate)
// ------------------------------------------------------------------------------------------------
__global__ void dot_fwd_kernel(const float* __restrict__ cand, const float* __restrict__ user, int B, int C, int D,
                               float* __restrict__ logits) {
    const int lane = threadIdx.x & 31;
    const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (wid >= B * C) return;
    const int b = wid / C;
    const float* cv = cand + static_cast<size_t>(wid) * D;
    const float* uv = user + static_cast<size_t>(b) * D;
    float a = 0.f;
    for (int c = lane; c < D; c += 32) a = fmaf(cv[c], uv[c], a);
    a = warp_sum(a);
    if (lane == 0) logits[wid] = a;
}
__global__ void dot_bwd_kernel(const float* __restrict__ cand, const float* __restrict__ user,
                               const float* __restrict__ dlogits, int B, int C, int D, float* __restrict__ dcand,
                               float* __restrict__ duser) {
    const int b = blockIdx.x;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        const float u = user[static_cast<size_t>(b) * D + c];
        float du = 0.f;
        for (int j = 0; j < C; ++j) {
            const float g = dlogits[b * C + j];
            dcand[(static_cast<size_t>(b) * C + j) * D + c] = g * u;
            du = fmaf(g, cand[(static_cast<size_t>(b) * C + j) * D + c], du);
        }
        duser[static_cast<size_t>(b) * D + c] = du;
    }
}
int dot_score_fwd(const float* cand, const float* user, int B, int C, int D, float* logits, cudaStream_t stream) {
    if (B * C == 0) return 0;
    ProfScope ps("dot_fwd", B, C, D, stream);
    dot_fwd_kernel<<<ceil_div(B * C * 32, 256), 256, 0, stream>>>(cand, user, B, C, D, logits);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}
int dot_score_bwd(const float* cand, const float* user, const float* dlogits, int B, int C, int D, float* dcand,
                  float* duser, cudaStream_t stream) {
    if (B == 0) return 0;
    ProfScope ps("dot_bwd", B, C, D, stream);
    dot_bwd_kernel<<<B, 128, 0, stream>>>(cand, user, dlogits, B, C, D, dcand, duser);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Precise user encoder (NRMS precise mode): the kernels that keep the history-level path at fp32 accuracy.
// The level is 4.6 % of the model's FLOPs (512 users x 50 news vectors), so plain CUDA-core arithmetic is affordable.
// ------------------------------------------------------------------------------------------------
// dst[e] += sum_s src[s * L + e] for e < L, s < n_seq (the gradient of a per-position addend shared by every sequence).  A CTA owns
// 32 consecutive e; warp w sums the sequences s = w (mod 8) in increasing order, the eight partials are added in warp order: the
// result is the same bits on every run (no atomics).
constexpr int kSeqSumWarps = 8;
__global__ void __launch_bounds__(32 * kSeqSumWarps) sum_over_seq_kernel(const float* __restrict__ src, long long n_seq, long long L,
                                                                        float* __restrict__ dst) {
    __shared__ float part[kSeqSumWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long e = blockIdx.x * 32ll + lane;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (e < L) {
        long long s = w;
        for (; s + 3 * kSeqSumWarps < n_seq; s += 4 * kSeqSumWarps) {
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[k] += src[(s + k * kSeqSumWarps) * L + e];
        }
        for (; s < n_seq; s += kSeqSumWarps) acc[0] += src[s * L + e];
    }
    part[w][lane] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
    __syncthreads();
    if (w == 0 && e < L) {
        float t = part[0][lane];
#pragma unroll
        for (int k = 1; k < kSeqSumWarps; ++k) t += part[k][lane];
        dst[e] += t;
    }
}
int sum_over_seq(const float* src, long long n_seq, long long L, float* dst, cudaStream_t stream) {
    if (n_seq == 0 || L == 0) return 0;
    NR_REQUIRE(L > 0 && (L + 31) / 32 < (1ll << 31), "sum_over_seq: L=%lld", L);
    ProfScope ps("sum_over_seq", static_cast<int>(n_seq), static_cast<int>(std::min<long long>(L, 1 << 30)), 0, stream);
    sum_over_seq_kernel<<<static_cast<unsigned>((L + 31) / 32), 32 * kSeqSumWarps, 0, stream>>>(src, n_seq, L, dst);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// fp32 multi-head self-attention core (multihead_self.py:15-23) on fp32 Q|K|V rows [n_seq*T][ld] (Q at column 0, K at d, V at
// 2d): one CTA per (sequence, head), thread i owns query row i (T <= 64): scores, exp-softmax with the +1e-8, P.V -- all in
// fp32 registers / shared memory.  The context leaves as bf16 hi + lo planes (pitch ldc, ones column at d in the hi plane).
constexpr int kF32MaxT = 64, kF32MaxDk = 32;
__global__ void __launch_bounds__(64) mhsa_f32_fwd_kernel(const float* __restrict__ qkv, int ld, int sec, int T, int heads, int dk,
                                                          __nv_bfloat16* __restrict__ c_hi, __nv_bfloat16* __restrict__ c_lo, int ldc) {
    __shared__ float sk[kF32MaxT][kF32MaxDk + 1], sv[kF32MaxT][kF32MaxDk + 1];
    const int seq = blockIdx.x / heads, h = blockIdx.x - seq * heads;
    const int d = heads * dk;
    const float* base = qkv + static_cast<size_t>(seq) * T * ld + h * dk;
    for (int i = threadIdx.x; i < T * dk; i += blockDim.x) {
        const int r = i / dk, c = i - r * dk;
        sk[r][c] = base[static_cast<size_t>(r) * ld + sec + c];
        sv[r][c] = base[static_cast<size_t>(r) * ld + 2 * sec + c];
    }
    __syncthreads();
    const int i = threadIdx.x;
    if (i >= T) return;
    float q[kF32MaxDk];
#pragma unroll
    for (int c = 0; c < kF32MaxDk; ++c) q[c] = c < dk ? base[static_cast<size_t>(i) * ld + c] : 0.f;
    const float rs = rsqrtf(static_cast<float>(dk));
    float s[kF32MaxT];
    float m = -INFINITY;
#pragma unroll 1
    for (int j = 0; j < T; ++j) {
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < kF32MaxDk; ++c) acc = fmaf(q[c], c < dk ? sk[j][c] : 0.f, acc);
        s[j] = acc * rs;
        m = fmaxf(m, s[j]);
    }
    float l = 0.f;
#pragma unroll 1
    for (int j = 0; j < T; ++j) {
        s[j] = __expf(s[j] - m);
        l += s[j];
    }
    const float inv = 1.f / (l + 1e-8f * __expf(-m));  // == exp(S) / (sum exp(S) + 1e-8)
    float o[kF32MaxDk];
#pragma unroll
    for (int c = 0; c < kF32MaxDk; ++c) o[c] = 0.f;
#pragma unroll 1
    for (int j = 0; j < T; ++j) {
        const float p = s[j] * inv;
#pragma unroll
        for (int c = 0; c < kF32MaxDk; ++c) o[c] = fmaf(p, c < dk ? sv[j][c] : 0.f, o[c]);
    }
    const size_t row = (static_cast<size_t>(seq) * T + i) * ldc;
#pragma unroll
    for (int c = 0; c < kF32MaxDk; ++c) {
        if (c < dk) {
            const __nv_bfloat16 hi = __float2bfloat16_rn(o[c]);
            c_hi[row + h * dk + c] = hi;
            c_lo[row + h * dk + c] = __float2bfloat16_rn(o[c] - __bfloat162float(hi));
        }
    }
    if (h == 0) {
        for (int c = d; c < ldc; ++c) {
            c_hi[row + c] = __float2bfloat16_rn(c == d ? 1.0f : 0.f);
            c_lo[row + c] = __float2bfloat16_rn(0.f);
        }
    }
}
// The same for d_k % 4 == 0 (the reference's 20): keys / values are read from shared memory as float4 (the scalar form above
// issues one ld.shared per FMA and is bound by it: 0.45 ms for the 512 x 15 history-level heads), the softmax runs online
// (one pass, no per-thread score array in local memory), exp(S)/(sum exp(S) + 1e-8) in its max-subtracted form.
template <int DK>
__global__ void __launch_bounds__(64) mhsa_f32_fwd_v4_kernel(const float* __restrict__ qkv, int ld, int sec, int T, int heads,
                                                             __nv_bfloat16* __restrict__ c_hi, __nv_bfloat16* __restrict__ c_lo, int ldc) {
    constexpr int V4 = DK / 4;
    __shared__ float4 sk[kF32MaxT][V4], sv[kF32MaxT][V4];
    const int seq = blockIdx.x / heads, h = blockIdx.x - seq * heads;
    const int d = heads * DK;
    const float* base = qkv + static_cast<size_t>(seq) * T * ld + h * DK;
    for (int i = threadIdx.x; i < T * V4; i += blockDim.x) {
        const int r = i / V4, c = i - r * V4;
        const float* kr = base + static_cast<size_t>(r) * ld + sec + 4 * c;
        const float* vr = base + static_cast<size_t>(r) * ld + 2 * sec + 4 * c;
        sk[r][c] = *reinterpret_cast<const float4*>(kr);  // 16-byte aligned: ld, sec multiples of 4, DK % 4 == 0
        sv[r][c] = *reinterpret_cast<const float4*>(vr);
    }
    __syncthreads();
    const int i = threadIdx.x;
    if (i >= T) return;
    float4 q[V4], o[V4];
    const float sc = rsqrtf(static_cast<float>(DK)) * 1.4426950408889634f;  // scores in the log2 domain
#pragma unroll
    for (int c = 0; c < V4; ++c) {
        const float4 qr = *reinterpret_cast<const float4*>(base + static_cast<size_t>(i) * ld + 4 * c);
        q[c] = make_float4(qr.x * sc, qr.y * sc, qr.z * sc, qr.w * sc);
        o[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float m = -INFINITY, l = 0.f;
#pragma unroll 2
    for (int j = 0; j < T; ++j) {
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int c = 0; c < V4; ++c) {
            const float4 k = sk[j][c];
            a0 = fmaf(q[c].x, k.x, a0); a1 = fmaf(q[c].y, k.y, a1);
            a0 = fmaf(q[c].z, k.z, a0); a1 = fmaf(q[c].w, k.w, a1);
        }
        const float sj = a0 + a1;
        const float mn = fmaxf(m, sj);
        const float r = exp2f(m - mn), pj = exp2f(sj - mn);  // first key: m = -inf -> r = 0
        l = fmaf(l, r, pj);
        m = mn;
#pragma unroll
        for (int c = 0; c < V4; ++c) {
            const float4 v = sv[j][c];
            o[c].x = fmaf(o[c].x, r, pj * v.x); o[c].y = fmaf(o[c].y, r, pj * v.y);
            o[c].z = fmaf(o[c].z, r, pj * v.z); o[c].w = fmaf(o[c].w, r, pj * v.w);
        }
    }
    const float inv = 1.f / (l + 1e-8f * exp2f(-m));  // == exp(S) / (sum exp(S) + 1e-8)
    const size_t row = (static_cast<size_t>(seq) * T + i) * ldc;
#pragma unroll
    for (int c = 0; c < V4; ++c) {
        const float ov[4] = {o[c].x * inv, o[c].y * inv, o[c].z * inv, o[c].w * inv};
        uint32_t hw[2], lw[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            hw[e] = pack_bf16x2(ov[2 * e], ov[2 * e + 1]);
            const float2 hf = unpack_bf16x2(hw[e]);
            lw[e] = pack_bf16x2(ov[2 * e] - hf.x, ov[2 * e + 1] - hf.y);
        }
        *reinterpret_cast<uint2*>(c_hi + row + h * DK + 4 * c) = make_uint2(hw[0], hw[1]);  // 8-byte aligned: ldc % 8 == 0, DK % 4 == 0
        *reinterpret_cast<uint2*>(c_lo + row + h * DK + 4 * c) = make_uint2(lw[0], lw[1]);
    }
    if (h == 0) {
        for (int c = d; c < ldc; ++c) {
            c_hi[row + c] = __float2bfloat16_rn(c == d ? 1.0f : 0.f);
            c_lo[row + c] = __float2bfloat16_rn(0.f);
        }
    }
}
int mhsa_f32_fwd(const float* qkv, int ld, int sec, long long n_seq, int T, int heads, int dk, void* c_hi, void* c_lo, int ldc,
                 cudaStream_t stream) {
    if (n_seq == 0) return 0;
    NR_REQUIRE(T >= 1 && T <= kF32MaxT && dk >= 1 && dk <= kF32MaxDk && ldc >= heads * dk + 1 && n_seq * heads < (1ll << 31),
               "mhsa_f32_fwd: T=%d dk=%d ldc=%d", T, dk, ldc);
    ProfScope ps("mhsa_f32_fwd", static_cast<int>(n_seq), T, heads * dk, stream);
    if (dk == 20 && ldc % 8 == 0 && ld % 4 == 0 && sec % 4 == 0) {
        mhsa_f32_fwd_v4_kernel<20><<<static_cast<int>(n_seq * heads), 64, 0, stream>>>(qkv, ld, sec, T, heads, static_cast<__nv_bfloat16*>(c_hi),
                                                                                       static_cast<__nv_bfloat16*>(c_lo), ldc);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    mhsa_f32_fwd_kernel<<<static_cast<int>(n_seq * heads), 64, 0, stream>>>(qkv, ld, sec, T, heads, dk, static_cast<__nv_bfloat16*>(c_hi),
                                                                           static_cast<__nv_bfloat16*>(c_lo), ldc);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// evaluation stage 3, batched (reference src/evaluate.py:245-265 scores ONE impression per get_prediction call and
// synchronises on .tolist() after each): scores[i] = news[cand[i]] . user[seg(i)] for the candidates of MANY impressions
// in one launch.  The news vectors stay in ONE device matrix (row = news index) instead of a Python dict of rows;
// seg_offsets[s] .. seg_offsets[s+1] delimit the candidates of impression s.  One warp per candidate, 16-byte loads.
// ------------------------------------------------------------------------------------------------
__global__ void segment_dot_kernel(const float* __restrict__ news, long long n_news, int D, const long long* __restrict__ cand,
                                   long long n_cand, const long long* __restrict__ seg_offsets, long long n_seg,
                                   const float* __restrict__ user, float* __restrict__ scores, int* __restrict__ bad_flag) {
    const int lane = threadIdx.x & 31;
    const long long w0 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
    const long long nw = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
    for (long long i = w0; i < n_cand; i += nw) {
        long long lo = 0, hi = n_seg;  // the impression of candidate i: last s with seg_offsets[s] <= i
        while (hi - lo > 1) {
            const long long mid = (lo + hi) >> 1;
            if (__ldg(seg_offsets + mid) <= i) lo = mid; else hi = mid;
        }
        long long nid = __ldg(cand + i);
        if (nid < 0 || nid >= n_news) {
            if (lane == 0) atomicExch(bad_flag, 1);
            nid = 0;
        }
        const float* nv = news + nid * D;
        const float* uv = user + lo * D;
        float acc = 0.f;
        if ((D & 3) == 0) {
            for (int c = lane * 4; c < D; c += 128) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(nv + c)), b = __ldg(reinterpret_cast<const float4*>(uv + c));
                acc = fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, fmaf(a.w, b.w, acc))));
            }
        } else {
            for (int c = lane; c < D; c += 32) acc = fmaf(nv[c], uv[c], acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) scores[i] = acc;
    }
}
int segment_dot(const float* news, long long n_news, int D, const long long* cand, long long n_cand, const long long* seg_offsets,
                long long n_seg, const float* user, float* scores, int* bad_flag, cudaStream_t stream) {
    if (n_cand == 0) return 0;
    ProfScope ps("segment_dot", static_cast<int>(n_cand), static_cast<int>(n_seg), D, stream);
    const int blocks = static_cast<int>(std::min<long long>((n_cand + 7) / 8, 148 * 16));
    segment_dot_kernel<<<blocks, 256, 0, stream>>>(news, n_news, D, cand, n_cand, seg_offsets, n_seg, user, scores, bad_flag);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// evaluation metrics (reference src/evaluate.py:160-168, 267-271: sklearn roc_auc_score + NumPy mrr / nDCG@5 / nDCG@10 once
// per impression in a process pool): {AUC, MRR, nDCG@5, nDCG@10} of EVERY impression in one launch.  One warp per
// impression; lane l owns candidates l, l+32, ... and counts, against every candidate of the impression, how many score
// higher (its 0-based place in the descending order, ties broken as the stable reading of argsort(s)[::-1]: the later
// candidate first) and, for a positive, how many negatives score lower / equal (Mann-Whitney AUC in integers).  The
// impression's (score, label) pairs are staged in a per-warp shared-memory chunk, chunk by chunk when it is longer.
// O(n^2) per impression: MIND impressions hold tens to a few hundred candidates.
// ------------------------------------------------------------------------------------------------
constexpr int kMetricWarps = 8, kMetricChunk = 512;
template <typename T>
__device__ __forceinline__ T warp_total(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// finite fp32 score -> int32 with the same order and -0 == +0.  The library builds with --use_fast_math (-ftz=true), under
// which fp32 comparisons treat subnormal scores as zero; integer keys keep every distinct finite score distinct.
__device__ __forceinline__ int score_key(float x) {
    const int b = __float_as_int(x) == static_cast<int>(0x80000000u) ? 0 : __float_as_int(x);
    return b < 0 ? b ^ 0x7fffffff : b;
}
__device__ __forceinline__ bool finite_score(float x) { return (__float_as_uint(x) & 0x7f800000u) != 0x7f800000u; }

// The place of every candidate of one impression of n candidates, for one warp: lane l owns candidates i = l, l+32, ... and
// calls visit(i, place_i, neg_lt_i, neg_eq_i) for each, where place_i = #{j : s_j > s_i} + #{j > i : s_j == s_i} and, with
// kLabels, neg_lt_i / neg_eq_i count the negatives (label 0) scoring below / level with it (0 without).  ck / cn are the
// warp's shared-memory chunk of kMetricChunk keys / negative marks; an impression longer than that is staged chunk by chunk.
// Ends with __syncwarp, so the warp may restage the chunk for its next impression.
template <bool kLabels, typename Visit>
__device__ __forceinline__ void impression_places(const float* sc, const unsigned char* lb, long long n, int lane, int* ck,
                                                  unsigned char* cn, Visit&& visit) {
    const bool one_chunk = n <= kMetricChunk;
    if (one_chunk) {
        for (int j = lane; j < n; j += 32) {
            ck[j] = score_key(__ldg(sc + j));
            if constexpr (kLabels) cn[j] = __ldg(lb + j) == 0;
        }
        __syncwarp();
    }
    for (long long i0 = 0; i0 < n; i0 += 32) {
        const long long i = i0 + lane;
        const bool own = i < n;
        const int ki = own ? score_key(__ldg(sc + i)) : 0;
        long long place = 0, neg_lt = 0, neg_eq = 0;  // place: #{higher} + #{level and later} = position in the descending order
        for (long long c0 = 0; c0 < n; c0 += kMetricChunk) {
            const int len = static_cast<int>(min(static_cast<long long>(kMetricChunk), n - c0));
            if (!one_chunk) {
                __syncwarp();
                for (int j = lane; j < len; j += 32) {
                    ck[j] = score_key(__ldg(sc + c0 + j));
                    if constexpr (kLabels) cn[j] = __ldg(lb + c0 + j) == 0;
                }
                __syncwarp();
            }
            const int after = static_cast<int>(max(-1ll, min(static_cast<long long>(len), i - c0)));  // chunk slots j > after are later than i
            int gt = 0, eq_after = 0, lt_neg = 0, eq_neg = 0;
            for (int j = 0; j < len; ++j) {
                const int kj = ck[j];
                const int eq = kj == ki;
                gt += kj > ki;
                eq_after += eq & (j > after);
                if constexpr (kLabels) {
                    const int neg = cn[j];
                    lt_neg += neg & (kj < ki);
                    eq_neg += neg & eq;
                }
            }
            place += gt + eq_after;
            neg_lt += lt_neg;
            neg_eq += eq_neg;
        }
        if (own) visit(i, place, neg_lt, neg_eq);
    }
    __syncwarp();  // the next impression restages this warp's chunk
}

__global__ void __launch_bounds__(kMetricWarps * 32) impression_metrics_kernel(const float* __restrict__ scores,
                                                                               const unsigned char* __restrict__ labels,
                                                                               const long long* __restrict__ seg_offsets, long long n_seg,
                                                                               double* __restrict__ metrics, int* __restrict__ bad_flag) {
    __shared__ int s_key[kMetricWarps][kMetricChunk];
    __shared__ unsigned char s_neg[kMetricWarps][kMetricChunk];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    int* const ck = s_key[wl];
    unsigned char* const cn = s_neg[wl];
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    const long long nw = static_cast<long long>(gridDim.x) * kMetricWarps;
    for (long long s = static_cast<long long>(blockIdx.x) * kMetricWarps + wl; s < n_seg; s += nw) {
        const long long b = __ldg(seg_offsets + s);
        const long long n = __ldg(seg_offsets + s + 1) - b;
        const float* const sc = scores + b;
        const unsigned char* const lb = labels + b;
        // pass 1: positives, non-finite scores, labels other than 0 / 1
        long long pos_cnt = 0;
        bool bad_score = false, bad_label = false;
        for (long long i = lane; i < n; i += 32) {
            const unsigned char l = __ldg(lb + i);
            pos_cnt += l == 1;
            bad_label |= l > 1;
            bad_score |= !finite_score(__ldg(sc + i));
        }
        const long long P = warp_total(pos_cnt);
        bad_label = __any_sync(0xffffffffu, bad_label);
        bad_score = __any_sync(0xffffffffu, bad_score);
        if (bad_label && lane == 0) atomicExch(bad_flag, 1);
        double* const out = metrics + 4 * s;
        if (bad_label || bad_score || P == 0) {  // sklearn raises (the reference catches it: NaN row); no positive: 0/0
            if (lane < 4) out[lane] = qnan;
            continue;
        }
        const long long N = n - P;
        // pass 2: lane l owns candidates i = l, l+32, ...; the comparison partners come from the shared-memory chunk
        unsigned long long auc2 = 0;  // sum over positives of 2 #{negatives below} + #{negatives level}
        double rr = 0.0, g5 = 0.0, g10 = 0.0;
        impression_places<true>(sc, lb, n, lane, ck, cn, [&](long long i, long long place, long long neg_lt, long long neg_eq) {
            if (__ldg(lb + i) == 1) {
                auc2 += static_cast<unsigned long long>(2 * neg_lt + neg_eq);
                rr += 1.0 / static_cast<double>(place + 1);
                const double g = place < 10 ? 1.0 / log2(static_cast<double>(place + 2)) : 0.0;
                g10 += g;
                g5 += place < 5 ? g : 0.0;
            }
        });
        auc2 = warp_total(auc2);
        rr = warp_total(rr);
        g5 = warp_total(g5);
        g10 = warp_total(g10);
        if (lane == 0) {
            double ideal5 = 0.0, ideal10 = 0.0;  // DCG of the ideal order: the P positives first
            for (int r = 0; r < 10 && r < P; ++r) {
                const double g = 1.0 / log2(static_cast<double>(r + 2));
                ideal10 += g;
                ideal5 += r < 5 ? g : 0.0;
            }
            // one class (no negative): roc_auc_score warns and returns NaN, MRR / nDCG stay defined
            out[0] = N > 0 ? static_cast<double>(auc2) / (2.0 * static_cast<double>(P) * static_cast<double>(N)) : qnan;
            out[1] = rr / static_cast<double>(P);
            out[2] = g5 / ideal5;
            out[3] = g10 / ideal10;
        }
    }
}
int impression_metrics(const float* scores, const unsigned char* labels, const long long* seg_offsets, long long n_seg, double* metrics,
                       int* bad_label_flag, cudaStream_t stream) {
    if (n_seg == 0) return 0;
    ProfScope ps("impression_metrics", static_cast<int>(std::min<long long>(n_seg, 1 << 30)), 0, 0, stream);
    const int blocks = static_cast<int>(std::min<long long>((n_seg + kMetricWarps - 1) / kMetricWarps, 148 * 16));
    impression_metrics_kernel<<<blocks, kMetricWarps * 32, 0, stream>>>(scores, labels, seg_offsets, n_seg, metrics, bad_label_flag);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// test-set predictions (the leaderboard's prediction.txt: one line "<impression_id> [r1,r2,...,rn]" per impression, r_i the
// 1-based rank of candidate i).  ranks[i] = place_i + 1 with the place nr_impression_metrics uses, so MRR / nDCG recomputed
// from the file agree with the evaluator; one warp per impression, the same shared-memory chunks.  An impression holding a
// non-finite score sets the flag and gets ranks 0: its order is undefined.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMetricWarps * 32) impression_ranks_kernel(const float* __restrict__ scores,
                                                                             const long long* __restrict__ seg_offsets, long long n_seg,
                                                                             int* __restrict__ ranks, int* __restrict__ bad_flag) {
    __shared__ int s_key[kMetricWarps][kMetricChunk];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const long long nw = static_cast<long long>(gridDim.x) * kMetricWarps;
    for (long long s = static_cast<long long>(blockIdx.x) * kMetricWarps + wl; s < n_seg; s += nw) {
        const long long b = __ldg(seg_offsets + s);
        const long long n = __ldg(seg_offsets + s + 1) - b;
        const float* const sc = scores + b;
        int* const rk = ranks + b;
        bool bad = false;
        for (long long i = lane; i < n; i += 32) bad |= !finite_score(__ldg(sc + i));
        if (__any_sync(0xffffffffu, bad)) {
            if (lane == 0) atomicExch(bad_flag, 1);
            for (long long i = lane; i < n; i += 32) rk[i] = 0;
            continue;
        }
        impression_places<false>(sc, nullptr, n, lane, s_key[wl], nullptr,
                                 [&](long long i, long long place, long long, long long) { rk[i] = static_cast<int>(place + 1); });
    }
}
int impression_ranks(const float* scores, const long long* seg_offsets, long long n_seg, int* ranks, int* bad_score_flag,
                     cudaStream_t stream) {
    if (n_seg == 0) return 0;
    ProfScope ps("impression_ranks", static_cast<int>(std::min<long long>(n_seg, 1 << 30)), 0, 0, stream);
    const int blocks = static_cast<int>(std::min<long long>((n_seg + kMetricWarps - 1) / kMetricWarps, 148 * 16));
    impression_ranks_kernel<<<blocks, kMetricWarps * 32, 0, stream>>>(scores, seg_offsets, n_seg, ranks, bad_score_flag);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// The text of the ranks: line s is "<ids[s]> [r_0,r_1,...,r_{n-1}]\n" (ids printed as unsigned decimal, ranks as unsigned
// decimal), its bytes at text[line_offsets[s] .. line_offsets[s+1]).  The lengths kernel and the text kernel count the same
// digits, so every line fills exactly its slot whatever the values.  One warp per impression; each lane writes the digits of
// its candidates at the position a warp scan of the digit counts gives, followed by ',' (or ']' after the last).
__device__ __forceinline__ int decimal_digits(unsigned long long v) {
    int d = 1;
    while (v >= 10ull) {
        v /= 10ull;
        ++d;
    }
    return d;
}
__device__ __forceinline__ void write_decimal(char* out, unsigned long long v, int digits) {
    for (int k = digits - 1; k >= 0; --k) {
        out[k] = static_cast<char>('0' + v % 10ull);
        v /= 10ull;
    }
}
constexpr int kTextWarps = 8;
__global__ void __launch_bounds__(kTextWarps * 32) prediction_line_lengths_kernel(const long long* __restrict__ ids,
                                                                                  const int* __restrict__ ranks,
                                                                                  const long long* __restrict__ seg_offsets,
                                                                                  long long n_seg, long long* __restrict__ lengths) {
    const int lane = threadIdx.x & 31;
    const long long nw = static_cast<long long>(gridDim.x) * kTextWarps;
    if (blockIdx.x == 0 && threadIdx.x == 0) lengths[n_seg] = 0;  // the scan's last entry becomes the total
    for (long long s = static_cast<long long>(blockIdx.x) * kTextWarps + (threadIdx.x >> 5); s < n_seg; s += nw) {
        const long long b = __ldg(seg_offsets + s);
        const long long n = __ldg(seg_offsets + s + 1) - b;
        long long body = 0;  // every rank's digits and the ',' or ']' after it
        for (long long i = lane; i < n; i += 32) body += decimal_digits(static_cast<unsigned>(__ldg(ranks + b + i))) + 1;
        body = warp_total(body);
        if (lane == 0)  // "<id> [" body "\n"; an empty impression is "<id> []\n"
            lengths[s] = decimal_digits(static_cast<unsigned long long>(__ldg(ids + s))) + 2 + body + (n == 0) + 1;
    }
}
__global__ void __launch_bounds__(kTextWarps * 32) prediction_text_kernel(const long long* __restrict__ ids, const int* __restrict__ ranks,
                                                                          const long long* __restrict__ seg_offsets, long long n_seg,
                                                                          const long long* __restrict__ line_offsets, char* __restrict__ text) {
    const int lane = threadIdx.x & 31;
    const long long nw = static_cast<long long>(gridDim.x) * kTextWarps;
    for (long long s = static_cast<long long>(blockIdx.x) * kTextWarps + (threadIdx.x >> 5); s < n_seg; s += nw) {
        const long long b = __ldg(seg_offsets + s);
        const long long n = __ldg(seg_offsets + s + 1) - b;
        char* const line = text + __ldg(line_offsets + s);
        const unsigned long long id = static_cast<unsigned long long>(__ldg(ids + s));
        const int id_digits = decimal_digits(id);
        if (lane == 0) {
            write_decimal(line, id, id_digits);
            line[id_digits] = ' ';
            line[id_digits + 1] = '[';
        }
        long long pos = id_digits + 2;
        for (long long i0 = 0; i0 < n; i0 += 32) {
            const long long i = i0 + lane;
            const unsigned r = i < n ? static_cast<unsigned>(__ldg(ranks + b + i)) : 0u;
            const int d = i < n ? decimal_digits(r) : 0;
            int incl = d + (i < n);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            if (i < n) {
                char* const at = line + pos + incl - d - 1;
                write_decimal(at, r, d);
                at[d] = i == n - 1 ? ']' : ',';
            }
            pos += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) {
            if (n == 0) line[pos++] = ']';
            line[pos] = '\n';
        }
    }
}
constexpr long long kMaxTextLines = (1ll << 31) - 1;  // the scan counts its n_seg + 1 entries in int32
static int text_blocks(long long n_seg) {
    return static_cast<int>(std::min<long long>((n_seg + kTextWarps - 1) / kTextWarps, 148 * 16));
}
long long prediction_scan_bytes(long long n_seg) {
    size_t bytes = 0;
    if (n_seg >= kMaxTextLines ||
        cub::DeviceScan::ExclusiveSum(nullptr, bytes, static_cast<long long*>(nullptr), static_cast<int>(n_seg + 1)) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    return static_cast<long long>(bytes);
}
int prediction_line_offsets(const long long* ids, const int* ranks, const long long* seg_offsets, long long n_seg, long long* line_offsets,
                            void* workspace, long long workspace_bytes, cudaStream_t stream) {
    NR_REQUIRE(n_seg < kMaxTextLines, "nr_prediction_line_offsets: n_seg=%lld lines (at most 2^31 - 2 per call)", n_seg);
    const long long need = prediction_scan_bytes(n_seg);
    NR_REQUIRE(need >= 0, "nr_prediction_line_offsets: scan workspace query failed for n_seg=%lld", n_seg);
    NR_REQUIRE(workspace_bytes >= need, "nr_prediction_line_offsets: workspace of %lld bytes, %lld needed", workspace_bytes, need);
    {
        ProfScope ps("prediction_line_lengths", static_cast<int>(std::min<long long>(n_seg, 1 << 30)), 0, 0, stream);
        prediction_line_lengths_kernel<<<std::max(1, text_blocks(n_seg)), kTextWarps * 32, 0, stream>>>(ids, ranks, seg_offsets, n_seg,
                                                                                                         line_offsets);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    size_t bytes = static_cast<size_t>(need);
    NR_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(workspace, bytes, line_offsets, static_cast<int>(n_seg + 1), stream));
    g_launches += 2;  // the scan's tile-state initialisation and the decoupled look-back scan
    return 0;
}
int prediction_text(const long long* ids, const int* ranks, const long long* seg_offsets, long long n_seg, const long long* line_offsets,
                    char* text, cudaStream_t stream) {
    if (n_seg == 0) return 0;
    ProfScope ps("prediction_text", static_cast<int>(std::min<long long>(n_seg, 1 << 30)), 0, 0, stream);
    prediction_text_kernel<<<text_blocks(n_seg), kTextWarps * 32, 0, stream>>>(ids, ranks, seg_offsets, n_seg, line_offsets, text);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Batch feed: the reference hands the model slot-major lists of per-slot (B, L) int64 tensors (default_collate over
// src/dataset.py:64-85; pinned by the DataLoader, src/train.py:165-171).  ONE launch reads the payload of every slot
// straight from page-locked host memory (unified addressing: the kernel's loads cross PCIe, no host staging copy, no
// per-slot cudaMemcpyAsync) and writes the impression-major block the encoders consume:
//   out[(b*H + h)*L + t] = clicked[h][b][t]            rows [0, B*H)
//   out[B*H*L + (b*C + c)*L + t] = candidates[c][b][t]  rows [B*H, B*(H+C))
// ------------------------------------------------------------------------------------------------
constexpr int kSlotTable = 64;
struct SlotTable {
    const long long* p[kSlotTable];
};
__global__ void __launch_bounds__(256) pack_slots_kernel(SlotTable tab, int n, int slot0, int H, int C, int B, int L, long long* __restrict__ out) {
    const long long per = static_cast<long long>(B) * L, total = per * n;
    for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += gridDim.x * 256ll) {
        const int sl = static_cast<int>(i / per);
        const long long rem = i - sl * per;
        const int b = static_cast<int>(rem / L), t = static_cast<int>(rem - static_cast<long long>(b) * L);
        const int s = slot0 + sl;
        const long long v = tab.p[sl][rem];
        const long long dst = s < H ? (static_cast<long long>(b) * H + s) * L + t
                                    : static_cast<long long>(B) * H * L + (static_cast<long long>(b) * C + (s - H)) * L + t;
        out[dst] = v;
    }
}
// 1 when every pointer is readable by a kernel on the current device (device / managed memory, or page-locked host memory
// whose device alias is the same address)
int slots_device_readable(const void* const* slots, int n) {
    for (int i = 0; i < n; ++i) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, slots[i]) != cudaSuccess) {
            cudaGetLastError();
            return 0;
        }
        if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) continue;
        if (at.type != cudaMemoryTypeHost || at.devicePointer != slots[i]) return 0;
    }
    return 1;
}
int pack_slots(const void* const* slots, int H, int C, int B, int L, long long* out, cudaStream_t stream) {
    const int n_slots = H + C;
    if (n_slots == 0 || B == 0 || L == 0) return 0;
    ProfScope ps("pack_slots", n_slots, B, L, stream);
    for (int s0 = 0; s0 < n_slots; s0 += kSlotTable) {
        SlotTable tab;
        const int n = std::min(kSlotTable, n_slots - s0);
        for (int i = 0; i < kSlotTable; ++i) tab.p[i] = static_cast<const long long*>(slots[s0 + std::min(i, n - 1)]);
        const long long total = static_cast<long long>(n) * B * L;
        const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 148 * 32));
        pack_slots_kernel<<<blocks, 256, 0, stream>>>(tab, n, s0, H, C, B, L, out);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Device feed: the news tables (int32 [n_news][width] per field), the behaviour table (int32 [R][H + C] news rows) and the
// per-row records live on the device; ONE launch writes the batch's impression-major int64 id block of every field (the
// layout pack_slots writes) and its records.  blockIdx.y is the field, y == n_fields the records (each output its own buffer:
// the trainer may change clicked_news_length in place while autograd holds user).  A thread item copies
// `vec` ids of one row: 4 (one 16-byte load, two 16-byte stores), 2 (an 8-byte load, one 16-byte store) or 1.
// ------------------------------------------------------------------------------------------------
struct FeedJob {
    const int* table;
    long long* out;
    int width, vec;
};
struct FeedJobs {
    FeedJob f[kFeedFields];
};
__global__ void __launch_bounds__(256) feed_gather_kernel(FeedJobs jobs, int n_fields, const int* __restrict__ beh, int H, int C,
                                                          FeedRecords rec, const long long* __restrict__ rows, int B) {
    const long long stride = gridDim.x * 256ll;
    if (static_cast<int>(blockIdx.y) == n_fields) {
        const int n_rec = 2 + C;
        for (long long i = blockIdx.x * 256ll + threadIdx.x; i < static_cast<long long>(n_rec) * B; i += stride) {
            const int k = static_cast<int>(i / B), b = static_cast<int>(i - static_cast<long long>(k) * B);
            long long* out = k == 0 ? rec.user : (k == 1 ? rec.length : rec.clicked);
            if (out) out[k < 2 ? b : i - 2ll * B] = rec.records[rows[b] * n_rec + k];
        }
        return;
    }
    const FeedJob j = jobs.f[blockIdx.y];
    const int per_row = j.width / j.vec;
    const long long n_browsed = static_cast<long long>(B) * H, total = static_cast<long long>(B) * (H + C) * per_row;
    for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += stride) {
        const long long r = i / per_row;
        const int k = static_cast<int>(i - r * per_row);
        long long b, s;
        if (r < n_browsed) {
            b = r / H;
            s = r - b * H;
        } else {
            b = (r - n_browsed) / C;
            s = H + (r - n_browsed - b * C);
        }
        const int news = beh[rows[b] * (H + C) + s];
        const int* src = j.table + static_cast<long long>(news) * j.width + k * j.vec;
        long long* dst = j.out + r * j.width + k * j.vec;
        if (j.vec == 4) {
            const int4 v = __ldg(reinterpret_cast<const int4*>(src));
            reinterpret_cast<longlong2*>(dst)[0] = make_longlong2(v.x, v.y);
            reinterpret_cast<longlong2*>(dst)[1] = make_longlong2(v.z, v.w);
        } else if (j.vec == 2) {
            const int2 v = __ldg(reinterpret_cast<const int2*>(src));
            *reinterpret_cast<longlong2*>(dst) = make_longlong2(v.x, v.y);
        } else {
            *dst = __ldg(src);
        }
    }
}
int feed_gather(const FeedField* fields, int n_fields, const int* behaviors, int H, int C, FeedRecords rec, const long long* rows, int B,
                cudaStream_t stream) {
    const int n_rec = rec.user || rec.length || rec.clicked ? 2 + C : 0;
    if (B == 0 || (n_fields == 0 && n_rec == 0)) return 0;
    const auto aligned = [](const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; };
    FeedJobs jobs{};
    long long most = static_cast<long long>(n_rec) * B;
    for (int f = 0; f < n_fields; ++f) {
        const FeedField& x = fields[f];
        const bool even = x.width % 2 == 0 && aligned(x.out, 16);
        const int vec = even && x.width % 4 == 0 && aligned(x.table, 16) ? 4 : (even && aligned(x.table, 8) ? 2 : 1);
        jobs.f[f] = {.table = x.table, .out = x.out, .width = x.width, .vec = vec};
        most = std::max(most, static_cast<long long>(B) * (H + C) * (x.width / vec));
    }
    ProfScope ps("feed_gather", n_fields, B, H + C, stream);
    const dim3 grid(static_cast<unsigned>(std::max<long long>(1, std::min<long long>((most + 255) / 256, num_sms() * 8ll))),
                    static_cast<unsigned>(n_fields + (n_rec > 0 ? 1 : 0)));
    feed_gather_kernel<<<grid, 256, 0, stream>>>(jobs, n_fields, behaviors, H, C, rec, rows, B);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Negative sampling (include/newsrec_b200.h, nr_sample_negatives): one warp per impression.  Pass 1 counts the positives P and
// negatives N with ballots; the impression's R = min(P, N / K) rows are its owned rows.  Pass 2 walks the candidates again:
// the p-th positive goes to row p, and a negative of ordinal j with sort key (h_j, j) -- one 64-bit integer, h_j in the high
// half -- finds its rank among the impression's N keys by counting the smaller ones; rank r < R*K lands in row r / K,
// candidate column 1 + r % K.  The keys are recomputed from j alone and staged in the warp's slice of shared memory: once per
// impression when N <= kNegTile (MIND's impressions), else tile by tile for every 32 candidates.  The work is O(N^2 / 32) per
// lane and integer only: the output is the same on every run and device.
// ------------------------------------------------------------------------------------------------
constexpr int kNegWarps = 8, kNegTile = 256;
constexpr unsigned long long kNegGolden = 0x9E3779B97F4A7C15ull;
// one link of the chained hash of (seed, epoch, impression, ordinal): x' = splitmix64's finaliser of (x ^ v) + golden ratio
__host__ __device__ inline unsigned long long neg_hash_step(unsigned long long x, unsigned long long v) {
    unsigned long long z = (x ^ v) + kNegGolden;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ inline unsigned long long neg_sort_key(unsigned long long imp_state, unsigned j) {
    return (neg_hash_step(imp_state, j) & 0xFFFFFFFF00000000ull) | j;
}
__global__ void __launch_bounds__(kNegWarps * 32) sample_negatives_kernel(const int* __restrict__ cand_rows, const unsigned char* __restrict__ labels,
                                                                          const long long* __restrict__ imp_offsets, long long n_imp,
                                                                          const long long* __restrict__ row_offsets, int K,
                                                                          unsigned long long epoch_state, int* __restrict__ beh, int H) {
    __shared__ unsigned long long keys_all[kNegWarps][kNegTile];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long* keys = keys_all[warp];
    const unsigned below = (1u << lane) - 1;
    const long long W = H + 1ll + K;
    for (long long i = blockIdx.x * static_cast<long long>(kNegWarps) + warp; i < n_imp; i += static_cast<long long>(gridDim.x) * kNegWarps) {
        const long long beg = imp_offsets[i], end = imp_offsets[i + 1];
        long long P = 0, N = 0;
        for (long long c0 = beg; c0 < end; c0 += 32) {
            const int l = c0 + lane < end ? labels[c0 + lane] : 255;
            P += __popc(__ballot_sync(~0u, l == 1));
            N += __popc(__ballot_sync(~0u, l == 0));
        }
        const long long row0 = row_offsets[i];
        const long long rows = std::min(std::min(P, N / K), row_offsets[i + 1] - row0);  // never past the owned rows
        if (rows <= 0) continue;
        const unsigned long long imp_state = neg_hash_step(epoch_state, static_cast<unsigned long long>(i));
        const long long taken = rows * K;
        const bool one_tile = N <= kNegTile;
        __syncwarp();  // the previous impression's compares are done with keys[]
        if (one_tile) {
            for (int t = lane; t < N; t += 32) keys[t] = neg_sort_key(imp_state, static_cast<unsigned>(t));
            __syncwarp();
        }
        long long p_seen = 0, n_seen = 0;
        for (long long c0 = beg; c0 < end; c0 += 32) {
            const long long c = c0 + lane;
            const int l = c < end ? labels[c] : 255;
            const unsigned pos = __ballot_sync(~0u, l == 1), neg = __ballot_sync(~0u, l == 0);
            if (l == 1) {
                const long long p = p_seen + __popc(pos & below);
                if (p < rows) beh[(row0 + p) * W + H] = cand_rows[c];
            }
            if (neg) {
                const unsigned long long mine = neg_sort_key(imp_state, static_cast<unsigned>(n_seen + __popc(neg & below)));
                long long rank = 0;
                for (long long t0 = 0; t0 < N; t0 += kNegTile) {
                    if (!one_tile) {
                        __syncwarp();
                        for (int t = lane; t < kNegTile && t0 + t < N; t += 32)
                            keys[t] = neg_sort_key(imp_state, static_cast<unsigned>(t0 + t));
                        __syncwarp();
                    }
                    const int n_t = static_cast<int>(std::min<long long>(kNegTile, N - t0));
                    int smaller = 0;
#pragma unroll 4
                    for (int t = 0; t < n_t; ++t) smaller += keys[t] < mine;
                    rank += smaller;
                }
                if (l == 0 && rank < taken) beh[(row0 + rank / K) * W + H + 1 + rank % K] = cand_rows[c];
            }
            p_seen += __popc(pos);
            n_seen += __popc(neg);
        }
    }
}
int sample_negatives(const int* cand_rows, const unsigned char* labels, const long long* imp_offsets, long long n_imp, const long long* row_offsets,
                     int K, unsigned long long seed, long long epoch, int* behaviors, int H, cudaStream_t stream) {
    if (n_imp == 0) return 0;
    const unsigned long long epoch_state = neg_hash_step(neg_hash_step(0, seed), static_cast<unsigned long long>(epoch));
    ProfScope ps("sample_negatives", static_cast<int>(std::min<long long>(n_imp, 1 << 30)), K, H, stream);
    const long long blocks = std::min<long long>((n_imp + kNegWarps - 1) / kNegWarps, num_sms() * 32ll);
    sample_negatives_kernel<<<static_cast<unsigned>(blocks), kNegWarps * 32, 0, stream>>>(cand_rows, labels, imp_offsets, n_imp, row_offsets, K,
                                                                                          epoch_state, behaviors, H);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace nr
