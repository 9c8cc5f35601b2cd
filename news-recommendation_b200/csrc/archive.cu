// Hi-Fi Ark after the news encoder, in fp32 on the CUDA cores (reference src/model/general/attention/self.py,
// src/model/HiFiArk/OMAP.py, src/model/general/attention/similarity.py, src/model/general/click_predictor/DNN.py).
//
// User side, one CTA per user, X = the H clicked-news vectors (H x F):
//   P1 = softmax_row(X X^T)   Y = P1 X + X   Q = softmax_over_h(Y W)   A = Q^T Y   (the archive, P x F)
// Scorer, one CTA per segment (a training user or an evaluation impression), for every candidate c of the segment:
//   w = softmax(A c)   u = w^T A   h = relu(W1 [c; u] + b1)   logit = w2 . h + b2
//
// Why fp32 and no tensor cores: the scores are unscaled dot products of F = 300-wide vectors (values near 18 at
// initialisation); rounding them to bf16 moves the softmax by percents.  The work is ~3 MFLOP per user each way.
//
// Training and evaluation call the same scorer kernel: the archive leaves the user kernel through global memory (P x F fp32
// per user, 3 MB at batch 512), so the scorer does not care whether its candidates are a user's 1 + K training candidates or
// the rows of an impression gathered from the news matrix.
//
// The backward kernels recompute the forward from their inputs instead of loading saved activations: at batch 512 Y alone
// would be 30 MB of HBM written and read again per step, while recomputing it is ~1/3 of the backward's arithmetic, which
// the fp32 pipes absorb.
//
// Weight gradients: every CTA writes its own partial row to the workspace and sum_over_seq adds the rows in a fixed order
// into the gradient (bit-identical across runs, no atomics).
//
// Column ownership: every "for (f = tid; f < F; f += kThreads)" loop hands column f to the same thread, so a thread may
// overwrite column f of a shared matrix after it alone has read it, without a barrier.
#include <algorithm>

#include "nr_common.cuh"
#include "nr_ops.h"

namespace nr {
namespace archive {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kMaxH = 50, kMaxF = 400, kMaxP = 32, kMaxHid = 32;

__host__ __device__ inline int pitch(int F) { return F + 4; }  // 16-byte rows, shifted by one bank quad per row

// sum over the block (every thread gets the result); red needs kWarps floats
__device__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[wp] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < kWarps; ++k) t += red[k];
    return t;
}

// dot of two F-long shared rows (F % 4 == 0, 16-byte aligned)
__device__ __forceinline__ float row_dot(const float* a, const float* b, int F) {
    float s0 = 0.f, s1 = 0.f;
    for (int f = 0; f < F; f += 4) {
        const float4 x = *reinterpret_cast<const float4*>(a + f), y = *reinterpret_cast<const float4*>(b + f);
        s0 = fmaf(x.x, y.x, fmaf(x.y, y.y, s0));
        s1 = fmaf(x.z, y.z, fmaf(x.w, y.w, s1));
    }
    return s0 + s1;
}

// in-place softmax of n values at v[0], v[stride], ... by one warp (max subtracted first, as F.softmax)
__device__ __forceinline__ void warp_softmax(float* v, int n, int stride) {
    const int lane = threadIdx.x & 31;
    float m = -INFINITY;
    for (int i = lane; i < n; i += 32) m = fmaxf(m, v[i * stride]);
    m = warp_max(m);
    float s = 0.f;
    for (int i = lane; i < n; i += 32) {
        const float e = __expf(v[i * stride] - m);
        v[i * stride] = e;
        s += e;
    }
    const float r = 1.f / warp_sum(s);
    for (int i = lane; i < n; i += 32) v[i * stride] *= r;
}

// ---- user side ------------------------------------------------------------------------------------------------------------
struct UserSmem {
    float *X, *Y, *P1, *Q, *DS, *DL, *G, *red;
    __device__ UserSmem(float* base, int H, int F, int P) {
        const int ld = pitch(F);
        X = base;                                  // max(H, P) rows: the backward puts dA (P x F) here
        Y = X + std::max(H, P) * ld;
        P1 = Y + H * ld;
        Q = P1 + H * H;
        DS = Q + H * P;
        DL = DS + H * H;
        G = DL + H * P;
        red = G + P * P;
    }
};
__host__ inline size_t user_smem_bytes(int H, int F, int P) {
    return sizeof(float) * (static_cast<size_t>(std::max(H, P) + H) * pitch(F) + 2 * H * H + 2 * H * P + P * P + kWarps);
}

// X (from hist), P1, Y and Q of user b in shared memory
__device__ void user_forward_core(const float* __restrict__ x, int H, int F, int P, const float* __restrict__ W, const UserSmem& s) {
    const int ld = pitch(F), tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
    for (int e = tid; e < H * (F / 4); e += kThreads) {
        const int h = e / (F / 4), f = (e - h * (F / 4)) * 4;
        *reinterpret_cast<float4*>(s.X + h * ld + f) = __ldg(reinterpret_cast<const float4*>(x + static_cast<size_t>(h) * F + f));
    }
    __syncthreads();
    for (int e = tid; e < H * H; e += kThreads) {  // S = X X^T (unscaled)
        const int i = e / H, j = e - i * H;
        s.P1[e] = row_dot(s.X + i * ld, s.X + j * ld, F);
    }
    __syncthreads();
    for (int i = wp; i < H; i += kWarps) warp_softmax(s.P1 + i * H, H, 1);
    __syncthreads();
    for (int f = tid; f < F; f += kThreads) {  // Y = P1 X + X, column f
        for (int h = 0; h < H; ++h) {
            float acc = s.X[h * ld + f];
            for (int i = 0; i < H; ++i) acc = fmaf(s.P1[h * H + i], s.X[i * ld + f], acc);
            s.Y[h * ld + f] = acc;
        }
    }
    __syncthreads();
    for (int e = wp; e < H * P; e += kWarps) {  // L = Y W, one warp per (h, p)
        const int h = e / P, p = e - h * P;
        float acc = 0.f;
        for (int f = lane; f < F; f += 32) acc = fmaf(s.Y[h * ld + f], __ldg(W + static_cast<size_t>(f) * P + p), acc);
        acc = warp_sum(acc);
        if (lane == 0) s.Q[e] = acc;
    }
    __syncthreads();
    for (int p = wp; p < P; p += kWarps) warp_softmax(s.Q + p, H, P);  // softmax over the history, per head
    __syncthreads();
}

// G = W^T W (P x P) into s.G; returns R = ||G * (1 - I)||_F to every thread
__device__ float regularizer(const float* __restrict__ W, int F, int P, const UserSmem& s) {
    float sq = 0.f;
    for (int e = threadIdx.x; e < P * P; e += kThreads) {
        const int p = e / P, q = e - p * P;
        float g = 0.f;
        for (int f = 0; f < F; ++f) g = fmaf(__ldg(W + static_cast<size_t>(f) * P + p), __ldg(W + static_cast<size_t>(f) * P + q), g);
        s.G[e] = g;
        if (p != q) sq = fmaf(g, g, sq);
    }
    return sqrtf(block_sum(sq, s.red));  // block_sum's barriers also publish s.G
}

__global__ void __launch_bounds__(kThreads, 1) archive_user_fwd_kernel(const float* __restrict__ hist, int H, int F, int P,
                                                                       const float* __restrict__ W, float* __restrict__ archive,
                                                                       float* __restrict__ reg_out) {
    extern __shared__ __align__(16) float smem[];
    const UserSmem s(smem, H, F, P);
    const int b = blockIdx.x, ld = pitch(F);
    user_forward_core(hist + static_cast<size_t>(b) * H * F, H, F, P, W, s);
    float* a = archive + static_cast<size_t>(b) * P * F;
    for (int f = threadIdx.x; f < F; f += kThreads) {  // A = Q^T Y
        for (int p = 0; p < P; ++p) {
            float acc = 0.f;
            for (int h = 0; h < H; ++h) acc = fmaf(s.Q[h * P + p], s.Y[h * ld + f], acc);
            a[static_cast<size_t>(p) * F + f] = acc;
        }
    }
    if (b == 0 && reg_out != nullptr) {
        const float r = regularizer(W, F, P, s);
        if (threadIdx.x == 0) *reg_out = r;
    }
}

// dhist (=) from darchive; dW partial row of user b into part[b][F][P]; block 0 adds dreg * dR/dW to its row
__global__ void __launch_bounds__(kThreads, 1) archive_user_bwd_kernel(const float* __restrict__ hist, int H, int F, int P,
                                                                       const float* __restrict__ W, const float* __restrict__ darchive,
                                                                       const float* __restrict__ dreg, float* __restrict__ dhist,
                                                                       float* __restrict__ part) {
    extern __shared__ __align__(16) float smem[];
    const UserSmem s(smem, H, F, P);
    const int b = blockIdx.x, ld = pitch(F), tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
    const float* x = hist + static_cast<size_t>(b) * H * F;
    float reg_scale = 0.f;  // dreg * 2 / R (0 when R == 0: torch's norm gradient at zero)
    if (b == 0 && dreg != nullptr) {
        const float r = regularizer(W, F, P, s);
        reg_scale = r > 0.f ? 2.f * __ldg(dreg) / r : 0.f;
    }
    user_forward_core(x, H, F, P, W, s);
    // dA -> the X rows (X is reloaded below)
    const float* da = darchive + static_cast<size_t>(b) * P * F;
    for (int e = tid; e < P * (F / 4); e += kThreads) {
        const int p = e / (F / 4), f = (e - p * (F / 4)) * 4;
        *reinterpret_cast<float4*>(s.X + p * ld + f) = __ldg(reinterpret_cast<const float4*>(da + static_cast<size_t>(p) * F + f));
    }
    __syncthreads();
    for (int e = tid; e < H * P; e += kThreads) {  // dQ[h][p] = dA_p . Y_h
        const int h = e / P, p = e - h * P;
        s.DL[e] = row_dot(s.X + p * ld, s.Y + h * ld, F);
    }
    __syncthreads();
    for (int p = wp; p < P; p += kWarps) {  // dL = Q * (dQ - sum_h Q dQ)  (softmax over h)
        float t = 0.f;
        for (int h = lane; h < H; h += 32) t = fmaf(s.Q[h * P + p], s.DL[h * P + p], t);
        t = warp_sum(t);
        for (int h = lane; h < H; h += 32) s.DL[h * P + p] = s.Q[h * P + p] * (s.DL[h * P + p] - t);
    }
    __syncthreads();
    float* prow = part + static_cast<size_t>(b) * F * P;
    for (int f = tid; f < F; f += kThreads) {
        // dW partial (Y^T dL), column f of Y read before this thread overwrites it with dY
        for (int p = 0; p < P; ++p) {
            float acc = 0.f;
            for (int h = 0; h < H; ++h) acc = fmaf(s.Y[h * ld + f], s.DL[h * P + p], acc);
            if (reg_scale != 0.f) {
                float g = 0.f;
                for (int q = 0; q < P; ++q)
                    if (q != p) g = fmaf(__ldg(W + static_cast<size_t>(f) * P + q), s.G[q * P + p], g);
                acc = fmaf(reg_scale, g, acc);
            }
            prow[static_cast<size_t>(f) * P + p] = acc;
        }
        // dY = Q dA + dL W^T (from the A path and the L path), then X back into column f
        for (int h = 0; h < H; ++h) {
            float acc = 0.f;
            for (int p = 0; p < P; ++p) {
                acc = fmaf(s.Q[h * P + p], s.X[p * ld + f], acc);
                acc = fmaf(s.DL[h * P + p], __ldg(W + static_cast<size_t>(f) * P + p), acc);
            }
            s.Y[h * ld + f] = acc;
        }
        for (int h = 0; h < H; ++h) s.X[h * ld + f] = __ldg(x + static_cast<size_t>(h) * F + f);
    }
    __syncthreads();
    for (int e = tid; e < H * H; e += kThreads) {  // dP1[i][j] = dY_i . X_j
        const int i = e / H, j = e - i * H;
        s.DS[e] = row_dot(s.Y + i * ld, s.X + j * ld, F);
    }
    __syncthreads();
    for (int i = wp; i < H; i += kWarps) {  // dS = P1 * (dP1 - rowsum(P1 dP1))
        float t = 0.f;
        for (int j = lane; j < H; j += 32) t = fmaf(s.P1[i * H + j], s.DS[i * H + j], t);
        t = warp_sum(t);
        for (int j = lane; j < H; j += 32) s.DS[i * H + j] = s.P1[i * H + j] * (s.DS[i * H + j] - t);
    }
    __syncthreads();
    float* dx = dhist + static_cast<size_t>(b) * H * F;
    for (int f = tid; f < F; f += kThreads) {  // dX = dY + P1^T dY + (dS + dS^T) X
        for (int h = 0; h < H; ++h) {
            float acc = s.Y[h * ld + f];
            for (int i = 0; i < H; ++i) {
                acc = fmaf(s.P1[i * H + h], s.Y[i * ld + f], acc);
                acc = fmaf(s.DS[h * H + i] + s.DS[i * H + h], s.X[i * ld + f], acc);
            }
            dx[static_cast<size_t>(h) * F + f] = acc;
        }
    }
}

// ---- scorer ---------------------------------------------------------------------------------------------------------------
struct ScoreSmem {
    float *A, *c, *u, *sc, *w, *h, *red;  // sc: scores (P), w: weights (P), h: hidden (Hd)
    float *dA, *dW1, *dz, *dw, *dh, *db1, *dw2;  // backward only
    __device__ ScoreSmem(float* base, int F, int P, int Hd, bool bwd) {
        const int ld = pitch(F);
        A = base;
        c = A + P * ld;
        u = c + F;
        sc = u + F;
        w = sc + kMaxP;
        h = w + kMaxP;
        red = h + kMaxHid;
        dA = red + kMaxHid;
        dW1 = dA + (bwd ? P * ld : 0);
        dz = dW1 + (bwd ? 2 * Hd * F : 0);
        dw = dz + (bwd ? 2 * F : 0);
        dh = dw + kMaxP;
        db1 = dh + kMaxHid;
        dw2 = db1 + kMaxHid;
    }
};
__host__ inline size_t score_smem_bytes(int F, int P, int Hd, bool bwd) {
    size_t n = static_cast<size_t>(P) * pitch(F) + 2 * F + 2 * kMaxP + 2 * kMaxHid;
    if (bwd) n += static_cast<size_t>(P) * pitch(F) + 2 * static_cast<size_t>(Hd) * F + 2 * F + kMaxP + 3 * kMaxHid + 4;
    return sizeof(float) * n;
}

// The one scoring routine of both scorer kernels: candidate row c (global) against the archive in s.A.  Leaves c, u, the
// similarity weights and the hidden layer in shared memory and returns the logit to every thread.
__device__ float score_candidate(const float* __restrict__ crow, int F, int P, const float* __restrict__ W1, const float* __restrict__ b1,
                                 int Hd, const float* __restrict__ w2, const float* __restrict__ b2, const ScoreSmem& s) {
    const int ld = pitch(F), tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
    __syncthreads();  // the previous candidate's readers of c / u / w / h are done
    for (int f = tid; f < F; f += kThreads) s.c[f] = __ldg(crow + f);
    __syncthreads();
    for (int p = wp; p < P; p += kWarps) {  // s = A c
        float acc = 0.f;
        for (int f = lane; f < F; f += 32) acc = fmaf(s.A[p * ld + f], s.c[f], acc);
        acc = warp_sum(acc);
        if (lane == 0) s.w[p] = acc;
    }
    __syncthreads();
    if (wp == 0) warp_softmax(s.w, P, 1);
    __syncthreads();
    for (int f = tid; f < F; f += kThreads) {  // u = w^T A
        float acc = 0.f;
        for (int p = 0; p < P; ++p) acc = fmaf(s.w[p], s.A[p * ld + f], acc);
        s.u[f] = acc;
    }
    __syncthreads();
    for (int k = wp; k < Hd; k += kWarps) {  // h = relu(W1 [c; u] + b1)
        const float* wr = W1 + static_cast<size_t>(k) * 2 * F;
        float acc = 0.f;
        for (int f = lane; f < F; f += 32) acc = fmaf(__ldg(wr + f), s.c[f], fmaf(__ldg(wr + F + f), s.u[f], acc));
        acc = warp_sum(acc);
        if (lane == 0) s.h[k] = fmaxf(acc + __ldg(b1 + k), 0.f);
    }
    __syncthreads();
    if (wp == 0) {
        float acc = lane < Hd ? __ldg(w2 + lane) * s.h[lane] : 0.f;
        acc = warp_sum(acc);
        if (lane == 0) s.red[0] = acc + __ldg(b2);
    }
    __syncthreads();
    return s.red[0];
}

__device__ __forceinline__ bool cand_row(const long long* cand, long long i, long long n_news, long long& row, int* bad) {
    row = cand != nullptr ? cand[i] : i;
    if (row < 0 || row >= n_news) {
        if (bad != nullptr && threadIdx.x == 0) *bad = 1;
        return false;
    }
    return true;
}

__device__ void load_archive(const float* __restrict__ a, int F, int P, float* dst) {
    const int ld = pitch(F);
    for (int e = threadIdx.x; e < P * (F / 4); e += kThreads) {
        const int p = e / (F / 4), f = (e - p * (F / 4)) * 4;
        *reinterpret_cast<float4*>(dst + p * ld + f) = __ldg(reinterpret_cast<const float4*>(a + static_cast<size_t>(p) * F + f));
    }
}

struct ScoreArgs {
    const float* news;
    long long n_news;
    int F;
    const long long *cand, *seg;
    const float* archive;
    int P;
    const float *W1, *b1;
    int Hd;
    const float *w2, *b2;
};

__global__ void __launch_bounds__(kThreads) archive_score_fwd_kernel(const __grid_constant__ ScoreArgs a, float* __restrict__ logits,
                                                                    int* __restrict__ bad) {
    extern __shared__ __align__(16) float smem[];
    const ScoreSmem s(smem, a.F, a.P, a.Hd, false);
    const long long seg = blockIdx.x;
    load_archive(a.archive + static_cast<size_t>(seg) * a.P * a.F, a.F, a.P, s.A);
    for (long long i = a.seg[seg]; i < a.seg[seg + 1]; ++i) {
        long long row;
        if (!cand_row(a.cand, i, a.n_news, row, bad)) {
            if (threadIdx.x == 0) logits[i] = __int_as_float(0x7fc00000);
            continue;
        }
        const float logit = score_candidate(a.news + static_cast<size_t>(row) * a.F, a.F, a.P, a.W1, a.b1, a.Hd, a.w2, a.b2, s);
        if (threadIdx.x == 0) logits[i] = logit;
    }
}

// dcand[i] (=) per candidate position, darchive[seg] (=), DNN partial rows of the segment (W1 | b1 | w2 | b2 sections)
__global__ void __launch_bounds__(kThreads, 1) archive_score_bwd_kernel(const __grid_constant__ ScoreArgs a, const float* __restrict__ dlogits,
                                                                       float* __restrict__ dcand, float* __restrict__ darchive,
                                                                       float* __restrict__ part_W1, float* __restrict__ part_b1,
                                                                       float* __restrict__ part_w2, float* __restrict__ part_b2) {
    extern __shared__ __align__(16) float smem[];
    const int F = a.F, P = a.P, Hd = a.Hd, ld = pitch(F), tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
    const ScoreSmem s(smem, F, P, Hd, true);
    const long long seg = blockIdx.x;
    load_archive(a.archive + static_cast<size_t>(seg) * P * F, F, P, s.A);
    for (int e = tid; e < P * ld; e += kThreads) s.dA[e] = 0.f;
    for (int e = tid; e < 2 * Hd * F; e += kThreads) s.dW1[e] = 0.f;
    if (tid < kMaxHid) s.db1[tid] = s.dw2[tid] = 0.f;
    float db2 = 0.f;  // thread 0
    for (long long i = a.seg[seg]; i < a.seg[seg + 1]; ++i) {
        long long row;
        if (!cand_row(a.cand, i, a.n_news, row, nullptr)) continue;
        score_candidate(a.news + static_cast<size_t>(row) * F, F, P, a.W1, a.b1, Hd, a.w2, a.b2, s);
        const float g = __ldg(dlogits + i);
        if (tid < Hd) {
            const float hk = s.h[tid];
            const float dh = hk > 0.f ? g * __ldg(a.w2 + tid) : 0.f;
            s.dh[tid] = dh;
            s.db1[tid] += dh;
            s.dw2[tid] = fmaf(g, hk, s.dw2[tid]);
        }
        if (tid == 0) db2 += g;
        __syncthreads();
        for (int j = tid; j < 2 * F; j += kThreads) {  // d[c; u] = W1^T dh ; dW1 += dh [c; u]^T
            const float z = j < F ? s.c[j] : s.u[j - F];
            float acc = 0.f;
            for (int k = 0; k < Hd; ++k) {
                acc = fmaf(s.dh[k], __ldg(a.W1 + static_cast<size_t>(k) * 2 * F + j), acc);
                s.dW1[k * 2 * F + j] = fmaf(s.dh[k], z, s.dW1[k * 2 * F + j]);
            }
            s.dz[j] = acc;
        }
        __syncthreads();
        for (int p = wp; p < P; p += kWarps) {  // dw_p = A_p . du
            float acc = 0.f;
            for (int f = lane; f < F; f += 32) acc = fmaf(s.A[p * ld + f], s.dz[F + f], acc);
            acc = warp_sum(acc);
            if (lane == 0) s.dw[p] = acc;
        }
        __syncthreads();
        if (wp == 0) {  // ds = w * (dw - sum w dw), in place
            const float wv = lane < P ? s.w[lane] : 0.f, dv = lane < P ? s.dw[lane] : 0.f;
            const float t = warp_sum(wv * dv);
            if (lane < P) s.dw[lane] = wv * (dv - t);
        }
        __syncthreads();
        float* dc = dcand + static_cast<size_t>(i) * F;
        for (int f = tid; f < F; f += kThreads) {
            const float du = s.dz[F + f], cf = s.c[f];
            float acc = s.dz[f];
            for (int p = 0; p < P; ++p) {
                const float ds = s.dw[p];
                acc = fmaf(ds, s.A[p * ld + f], acc);
                s.dA[p * ld + f] = fmaf(s.w[p], du, fmaf(ds, cf, s.dA[p * ld + f]));
            }
            dc[f] = acc;
        }
    }
    __syncthreads();
    float* da = darchive + static_cast<size_t>(seg) * P * F;
    for (int e = tid; e < P * F; e += kThreads) {
        const int p = e / F, f = e - p * F;
        da[e] = s.dA[p * ld + f];
    }
    float* pw = part_W1 + static_cast<size_t>(seg) * 2 * Hd * F;
    for (int e = tid; e < 2 * Hd * F; e += kThreads) pw[e] = s.dW1[e];
    if (tid < Hd) {
        part_b1[seg * Hd + tid] = s.db1[tid];
        part_w2[seg * Hd + tid] = s.dw2[tid];
    }
    if (tid == 0) part_b2[seg] = db2;
}

// ---- DKN history attention (reference src/model/DKN/attention.py): user = sum_j softmax_j(beta . h_j) h_j -------------------
// beta = W1[:, F:]^T w2 (the candidate half and both biases cancel in the softmax, include/newsrec_b200.h).  One CTA per user;
// shared memory: beta, and the user's H scores / weights and their gradients.
namespace dkn {
constexpr int kMaxH = 64, kMaxF = 512, kMaxHid = 32;

// beta (F) from the history half of W1 (hidden x 2F) and w2
__device__ void load_beta(const float* __restrict__ W1, int Hd, const float* __restrict__ w2, int F, float* beta) {
    for (int f = threadIdx.x; f < F; f += kThreads) {
        float acc = 0.f;
        for (int k = 0; k < Hd; ++k) acc = fmaf(__ldg(W1 + static_cast<size_t>(k) * 2 * F + F + f), __ldg(w2 + k), acc);
        beta[f] = acc;
    }
}

// wt[j] = softmax_j(beta . x_j) for the H rows of x (F wide)
__device__ void history_weights(const float* __restrict__ x, int H, int F, const float* beta, float* wt) {
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    __syncthreads();  // beta
    for (int j = wp; j < H; j += kWarps) {
        float acc = 0.f;
        for (int f = lane; f < F; f += 32) acc = fmaf(__ldg(x + static_cast<size_t>(j) * F + f), beta[f], acc);
        acc = warp_sum(acc);
        if (lane == 0) wt[j] = acc;
    }
    __syncthreads();
    if (wp == 0) warp_softmax(wt, H, 1);
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads) dkn_user_fwd_kernel(const float* __restrict__ hist, int H, int F, const float* __restrict__ W1,
                                                                int Hd, const float* __restrict__ w2, float* __restrict__ user) {
    __shared__ float beta[kMaxF], wt[kMaxH];
    const float* x = hist + static_cast<size_t>(blockIdx.x) * H * F;
    load_beta(W1, Hd, w2, F, beta);
    history_weights(x, H, F, beta, wt);
    for (int f = threadIdx.x; f < F; f += kThreads) {
        float acc = 0.f;
        for (int j = 0; j < H; ++j) acc = fmaf(wt[j], __ldg(x + static_cast<size_t>(j) * F + f), acc);
        user[static_cast<size_t>(blockIdx.x) * F + f] = acc;
    }
}

// dw_j = du . x_j ; ds_j = w_j (dw_j - sum w dw) ; dx_j = w_j du + ds_j beta ; part[b] = dbeta_b = sum_j ds_j x_j
__global__ void __launch_bounds__(kThreads) dkn_user_bwd_kernel(const float* __restrict__ hist, int H, int F, const float* __restrict__ W1,
                                                                int Hd, const float* __restrict__ w2, const float* __restrict__ duser,
                                                                float* __restrict__ dhist, float* __restrict__ part) {
    __shared__ float beta[kMaxF], du[kMaxF], wt[kMaxH], ds[kMaxH];
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const size_t b = blockIdx.x;
    const float* x = hist + b * H * F;
    load_beta(W1, Hd, w2, F, beta);
    for (int f = threadIdx.x; f < F; f += kThreads) du[f] = __ldg(duser + b * F + f);
    history_weights(x, H, F, beta, wt);
    for (int j = wp; j < H; j += kWarps) {
        float acc = 0.f;
        for (int f = lane; f < F; f += 32) acc = fmaf(__ldg(x + static_cast<size_t>(j) * F + f), du[f], acc);
        acc = warp_sum(acc);
        if (lane == 0) ds[j] = acc;
    }
    __syncthreads();
    if (wp == 0) {
        float t = 0.f;
        for (int j = lane; j < H; j += 32) t = fmaf(wt[j], ds[j], t);
        t = warp_sum(t);
        for (int j = lane; j < H; j += 32) ds[j] = wt[j] * (ds[j] - t);
    }
    __syncthreads();
    for (int f = threadIdx.x; f < F; f += kThreads) {
        const float uf = du[f], bf = beta[f];
        float db = 0.f;
        for (int j = 0; j < H; ++j) {
            const float xj = __ldg(x + static_cast<size_t>(j) * F + f);
            dhist[b * H * F + static_cast<size_t>(j) * F + f] = fmaf(wt[j], uf, ds[j] * bf);
            db = fmaf(ds[j], xj, db);
        }
        part[b * F + f] = db;
    }
}

// dW1[k][F + f] += w2[k] dbeta[f] ; dw2[k] += sum_f W1[k][F + f] dbeta[f]   (one CTA; dbeta is the ordered sum of the partial rows)
__global__ void __launch_bounds__(kThreads) dkn_beta_bwd_kernel(int F, const float* __restrict__ W1, int Hd, const float* __restrict__ w2,
                                                                const float* __restrict__ dbeta, float* __restrict__ dW1,
                                                                float* __restrict__ dw2) {
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    for (int e = threadIdx.x; e < Hd * F; e += kThreads) {
        const int k = e / F, f = e - k * F;
        dW1[static_cast<size_t>(k) * 2 * F + F + f] += __ldg(w2 + k) * dbeta[f];
    }
    for (int k = wp; k < Hd; k += kWarps) {
        float acc = 0.f;
        for (int f = lane; f < F; f += 32) acc = fmaf(__ldg(W1 + static_cast<size_t>(k) * 2 * F + F + f), dbeta[f], acc);
        acc = warp_sum(acc);
        if (lane == 0) dw2[k] += acc;
    }
}
}  // namespace dkn

}  // namespace archive

using namespace archive;

static int set_smem(const void* kernel, size_t bytes) {
    NR_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
    return 0;
}

static int archive_user_fwd(const float* hist, long long B, int H, int F, int P, const float* W, float* archive, float* reg_out,
                     cudaStream_t stream) {
    const size_t smem = user_smem_bytes(H, F, P);
    NR_PROPAGATE(set_smem(reinterpret_cast<const void*>(archive_user_fwd_kernel), smem));
    ProfScope ps("archive_user_fwd", static_cast<int>(B), H, F, stream);
    archive_user_fwd_kernel<<<static_cast<unsigned>(B), kThreads, smem, stream>>>(hist, H, F, P, W, archive, reg_out);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int archive_user_bwd(const float* hist, long long B, int H, int F, int P, const float* W, const float* darchive, const float* dreg,
                     float* dhist, float* part, cudaStream_t stream) {
    const size_t smem = user_smem_bytes(H, F, P);
    NR_PROPAGATE(set_smem(reinterpret_cast<const void*>(archive_user_bwd_kernel), smem));
    ProfScope ps("archive_user_bwd", static_cast<int>(B), H, F, stream);
    archive_user_bwd_kernel<<<static_cast<unsigned>(B), kThreads, smem, stream>>>(hist, H, F, P, W, darchive, dreg, dhist, part);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int archive_score_fwd(const ScoreArgs& a, long long n_seg, float* logits, int* bad, cudaStream_t stream) {
    const size_t smem = score_smem_bytes(a.F, a.P, a.Hd, false);
    NR_PROPAGATE(set_smem(reinterpret_cast<const void*>(archive_score_fwd_kernel), smem));
    ProfScope ps("archive_score_fwd", static_cast<int>(n_seg), a.P, a.F, stream);
    archive_score_fwd_kernel<<<static_cast<unsigned>(n_seg), kThreads, smem, stream>>>(a, logits, bad);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int archive_score_bwd(const ScoreArgs& a, long long n_seg, const float* dlogits, float* dcand, float* darchive, float* part_W1,
                      float* part_b1, float* part_w2, float* part_b2, cudaStream_t stream) {
    const size_t smem = score_smem_bytes(a.F, a.P, a.Hd, true);
    NR_PROPAGATE(set_smem(reinterpret_cast<const void*>(archive_score_bwd_kernel), smem));
    ProfScope ps("archive_score_bwd", static_cast<int>(n_seg), a.P, a.F, stream);
    archive_score_bwd_kernel<<<static_cast<unsigned>(n_seg), kThreads, smem, stream>>>(a, dlogits, dcand, darchive, part_W1, part_b1,
                                                                                     part_w2, part_b2);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---- C ABI ------------------------------------------------------------------------------------------------------------------
// Shapes outside the supported bounds return kArchiveBounds (-2) before any launch; null operands and other argument errors -1.
constexpr int kArchiveBounds = -2;
#define ARCHIVE_BOUNDS(cond, ...)           \
    do {                                    \
        if (!(cond)) {                      \
            nr::set_error(__VA_ARGS__);     \
            return kArchiveBounds;          \
        }                                   \
    } while (0)

static int check_user(long long B, int H, int F, int P) {
    ARCHIVE_BOUNDS(B >= 0 && B < (1ll << 31) && H >= 1 && H <= kMaxH && F >= 4 && F <= kMaxF && F % 4 == 0 && P >= 1 && P <= kMaxP,
                   "archive user: shape outside the supported bounds (B=%lld H=%d F=%d P=%d; need 1 <= H <= %d, 4 <= F <= %d with F %% 4 == 0, "
                   "1 <= P <= %d)", B, H, F, P, kMaxH, kMaxF, kMaxP);
    return 0;
}
static int check_score(long long n_cand, long long n_seg, int F, int P, int Hd) {
    ARCHIVE_BOUNDS(n_cand >= 0 && n_seg >= 0 && n_seg < (1ll << 31) && F >= 4 && F <= kMaxF && F % 4 == 0 && P >= 1 && P <= kMaxP &&
                       Hd >= 1 && Hd <= kMaxHid,
                   "archive scorer: shape outside the supported bounds (n_seg=%lld F=%d P=%d hidden=%d; need 4 <= F <= %d with F %% 4 == 0, "
                   "1 <= P <= %d, 1 <= hidden <= %d)", n_seg, F, P, Hd, kMaxF, kMaxP, kMaxHid);
    return 0;
}
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

extern "C" {

int nr_archive_user_fwd(const float* hist, long long B, int H, int F, int P, const float* W, float* archive, float* reg_out, void* stream) {
    NR_PROPAGATE(check_user(B, H, F, P));
    NR_REQUIRE(hist && W && archive, "nr_archive_user_fwd: null operand");
    NR_REQUIRE(aligned16(hist) && aligned16(archive), "nr_archive_user_fwd: hist and archive must be 16-byte aligned");
    if (B == 0) return 0;
    prof_context("archive.fwd");
    return archive_user_fwd(hist, B, H, F, P, W, archive, reg_out, as_stream(stream));
}

long long nr_archive_user_bwd_workspace(long long B, int F, int P) { return align256(B * F * P * static_cast<long long>(sizeof(float))) + 256; }

int nr_archive_user_bwd(const float* hist, long long B, int H, int F, int P, const float* W, const float* darchive, const float* dreg,
                        float* dhist, float* dW, void* workspace, long long workspace_bytes, void* stream) {
    NR_PROPAGATE(check_user(B, H, F, P));
    NR_REQUIRE(hist && W && darchive && dhist && dW && workspace, "nr_archive_user_bwd: null operand");
    NR_REQUIRE(aligned16(hist) && aligned16(darchive), "nr_archive_user_bwd: hist and darchive must be 16-byte aligned");
    NR_REQUIRE(workspace_bytes >= nr_archive_user_bwd_workspace(B, F, P), "nr_archive_user_bwd: workspace too small");
    if (B == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    prof_context("archive.bwd");
    float* part = static_cast<float*>(workspace);
    NR_PROPAGATE(archive_user_bwd(hist, B, H, F, P, W, darchive, dreg, dhist, part, st));
    return sum_over_seq(part, B, static_cast<long long>(F) * P, dW, st);
}

int nr_archive_score_fwd(const float* news, long long n_news, int F, const long long* cand, long long n_cand, const long long* seg_offsets,
                         long long n_seg, const float* archive, int P, const float* W1, const float* b1, int Hd, const float* w2,
                         const float* b2, float* logits, int* bad_id_flag, void* stream) {
    NR_PROPAGATE(check_score(n_cand, n_seg, F, P, Hd));
    NR_REQUIRE(news && seg_offsets && archive && W1 && b1 && w2 && b2 && logits, "nr_archive_score_fwd: null operand");
    NR_REQUIRE(cand == nullptr || bad_id_flag != nullptr, "nr_archive_score_fwd: null operand (bad_id_flag with a candidate index)");
    NR_REQUIRE(aligned16(archive), "nr_archive_score_fwd: archive must be 16-byte aligned");
    if (n_seg == 0) return 0;
    prof_context("archive.fwd");
    const ScoreArgs a{news, n_news, F, cand, seg_offsets, archive, P, W1, b1, Hd, w2, b2};
    return archive_score_fwd(a, n_seg, logits, bad_id_flag, as_stream(stream));
}

long long nr_archive_score_bwd_workspace(long long n_seg, int F, int Hd) {
    WorkspaceLayout ws{nullptr};
    ws.take<float>(n_seg * 2 * Hd * F);
    ws.take<float>(n_seg * Hd);
    ws.take<float>(n_seg * Hd);
    ws.take<float>(n_seg);
    return ws.bytes();
}

int nr_archive_score_bwd(const float* news, long long n_news, int F, const long long* cand, long long n_cand, const long long* seg_offsets,
                         long long n_seg, const float* archive, int P, const float* W1, const float* b1, int Hd, const float* w2,
                         const float* b2, const float* dlogits, float* dcand, float* darchive, float* dW1, float* db1, float* dw2,
                         float* db2, void* workspace, long long workspace_bytes, void* stream) {
    NR_PROPAGATE(check_score(n_cand, n_seg, F, P, Hd));
    NR_REQUIRE(news && seg_offsets && archive && W1 && b1 && w2 && b2 && dlogits && dcand && darchive && dW1 && db1 && dw2 && db2 &&
                   workspace, "nr_archive_score_bwd: null operand");
    NR_REQUIRE(aligned16(archive), "nr_archive_score_bwd: archive must be 16-byte aligned");
    NR_REQUIRE(workspace_bytes >= nr_archive_score_bwd_workspace(n_seg, F, Hd), "nr_archive_score_bwd: workspace too small");
    if (n_seg == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    prof_context("archive.bwd");
    WorkspaceLayout ws{static_cast<char*>(workspace)};
    float* pW1 = ws.take<float>(n_seg * 2 * Hd * F);
    float* pb1 = ws.take<float>(n_seg * Hd);
    float* pw2 = ws.take<float>(n_seg * Hd);
    float* pb2 = ws.take<float>(n_seg);
    const ScoreArgs a{news, n_news, F, cand, seg_offsets, archive, P, W1, b1, Hd, w2, b2};
    NR_PROPAGATE(archive_score_bwd(a, n_seg, dlogits, dcand, darchive, pW1, pb1, pw2, pb2, st));
    NR_PROPAGATE(sum_over_seq(pW1, n_seg, 2ll * Hd * F, dW1, st));
    NR_PROPAGATE(sum_over_seq(pb1, n_seg, Hd, db1, st));
    NR_PROPAGATE(sum_over_seq(pw2, n_seg, Hd, dw2, st));
    return sum_over_seq(pb2, n_seg, 1, db2, st);
}

static int check_dkn_user(long long B, int H, int F, int Hd) {
    ARCHIVE_BOUNDS(B >= 0 && B < (1ll << 31) && H >= 1 && H <= dkn::kMaxH && F >= 1 && F <= dkn::kMaxF && Hd >= 1 && Hd <= dkn::kMaxHid,
                   "dkn user: shape outside the supported bounds (B=%lld H=%d F=%d hidden=%d; need 1 <= H <= %d, 1 <= F <= %d, "
                   "1 <= hidden <= %d)", B, H, F, Hd, dkn::kMaxH, dkn::kMaxF, dkn::kMaxHid);
    return 0;
}

int nr_dkn_user_fwd(const float* hist, long long B, int H, int F, const float* W1, int Hd, const float* w2, float* user, void* stream) {
    NR_PROPAGATE(check_dkn_user(B, H, F, Hd));
    NR_REQUIRE(hist && W1 && w2 && user, "nr_dkn_user_fwd: null operand");
    if (B == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    prof_context("dkn.fwd");
    ProfScope ps("dkn_user_fwd", static_cast<int>(B), H, F, st);
    dkn::dkn_user_fwd_kernel<<<static_cast<unsigned>(B), kThreads, 0, st>>>(hist, H, F, W1, Hd, w2, user);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

long long nr_dkn_user_bwd_workspace(long long B, int F) {
    WorkspaceLayout ws{nullptr};
    ws.take<float>(B * F);
    ws.take<float>(F);
    return ws.bytes();
}

int nr_dkn_user_bwd(const float* hist, long long B, int H, int F, const float* W1, int Hd, const float* w2, const float* duser, float* dhist,
                    float* dW1, float* dw2, void* workspace, long long workspace_bytes, void* stream) {
    NR_PROPAGATE(check_dkn_user(B, H, F, Hd));
    NR_REQUIRE(hist && W1 && w2 && duser && dhist && dW1 && dw2 && workspace, "nr_dkn_user_bwd: null operand");
    NR_REQUIRE(workspace_bytes >= nr_dkn_user_bwd_workspace(B, F), "nr_dkn_user_bwd: workspace too small");
    if (B == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    prof_context("dkn.bwd");
    WorkspaceLayout ws{static_cast<char*>(workspace)};
    float* part = ws.take<float>(B * F);
    float* dbeta = ws.take<float>(F);
    {
        ProfScope ps("dkn_user_bwd", static_cast<int>(B), H, F, st);
        dkn::dkn_user_bwd_kernel<<<static_cast<unsigned>(B), kThreads, 0, st>>>(hist, H, F, W1, Hd, w2, duser, dhist, part);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
    }
    NR_CHECK_CUDA(cudaMemsetAsync(dbeta, 0, sizeof(float) * F, st));
    NR_PROPAGATE(sum_over_seq(part, B, F, dbeta, st));
    ProfScope ps("dkn_beta_bwd", static_cast<int>(B), Hd, F, st);
    dkn::dkn_beta_bwd_kernel<<<1, kThreads, 0, st>>>(F, W1, Hd, w2, dbeta, dW1, dw2);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"

}  // namespace nr
