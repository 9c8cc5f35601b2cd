// Persistent recurrence of the LSTUR user encoder's GRU (reference src/model/LSTUR/user_encoder.py:27-45), forward:
// ONE cooperative launch runs all S time steps instead of 3 launches per step.
//
//   gh_t = h_{t-1} . W_hh^T + b_hh            [B x Hd] x [Hd x 3Hd]   (wgmma, bf16 operands, fp32 accumulate)
//   r = sig(gi_r + gh_r), z = sig(gi_z + gh_z), n = tanh(gi_n + r * gh_n), h_t = (1 - z) n + z h_{t-1}   for t < len[b]
//
// Decomposition: users in 128-row tiles (m) x hidden units in slices of 32 (s); CTA (m, s) keeps its 96 weight rows
// (32 units x gates r, z, n; 12 KB per 64 columns of Hd, SWIZZLE_128B K-major) resident in shared memory for the whole launch
// and the fp32 hidden state of its 128 x 32 block in REGISTERS.  Per step it streams the bf16 h_{t-1} rows of its tile (all
// Hd columns, written by the slice CTAs of the same row tile) through a 2-stage TMA ring; the four gate warps (one
// warpgroup) issue two m64n96 wgmmas per k-step and run the gates straight on the accumulator fragments (the r, z and n
// columns of a unit sit in the same thread).  Up to Hd = 1024 (16 k-chunks of resident weights).  Steps are separated by a release/acquire counter barrier per ROW TILE (only the slices of one tile exchange
// data).  The launch is cooperative (all CTAs resident) -- row_tiles * slices <= SM count is checked by the host.
// Saved for the (per-step) backward: gh (fp32), hs (fp32), hb (bf16 operand rows with the ones column), as before.
#include <algorithm>
#include <cstring>

#define NR_WATCHDOG_SYMBOL g_gru_dev_error
#include "nr_fused.cuh"
#include "nr_ops.h"

namespace nr {

int read_attn_device_error(int* out4);
int read_gru_device_error(int* out4) {
    const int rc = static_cast<int>(cudaMemcpyFromSymbol(out4, fused::g_gru_dev_error, sizeof(int) * 4));
    if (rc != 0 || out4[0] != 0) return rc;
    return read_attn_device_error(out4);  // the title-level attention kernel keeps its own record (attn_title.cu)
}

namespace gru {

using namespace fused;

constexpr int kThreads = 5 * 32;   // 4 gate warps (one warpgroup: wgmma + gates) + TMA producer
constexpr int kU = 32;             // hidden units per slice
constexpr int kN = 3 * kU;         // MMA N: gates r | z | n of the slice
constexpr int kWChunk = kN * 128;  // one 64-column k-chunk of the resident weight slice
constexpr int kAStage = 128 * 128;
constexpr int kAStages = 2;

struct Params {
    int B, S, Hd, ldh, ldg;
    int slices, k_chunks;
    const float* gi;         // [B*S][ldg]  rows b*S + t
    const float* bhh;        // [3Hd]
    const float* h0;         // [B][Hd]
    const long long* len;    // [B]
    float* gh;               // [S][B][ldg]
    float* hs;               // [S+1][B][Hd]   hs[0] = h0 (filled by the caller)
    __nv_bfloat16* hb;       // [S+1][B][ldh]  hb[0] = bf16(h0) + ones column (filled by the caller)
    float* out;              // [B][Hd]
    unsigned int* bar;       // [row tiles] step barrier counters, zero on entry
};

__device__ __forceinline__ unsigned int ld_acquire(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release(unsigned int* p) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}

__global__ void __launch_bounds__(kThreads, 1) gru_fwd_persistent_kernel(const __grid_constant__ CUtensorMap tmH,
                                                                         const __grid_constant__ CUtensorMap tmW, const Params p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sW = base;
    uint8_t* sA = sW + p.k_chunks * kWChunk;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sA + kAStages * kAStage);
    uint64_t* wfull = bars;            // resident weights landed
    uint64_t* afull = bars + 1;        // [kAStages]
    uint64_t* aempty = bars + 1 + kAStages;
    float* sBias = reinterpret_cast<float*>(bars + 16);      // [3][kU] b_hh of this slice (zero for units that do not exist); 16-byte aligned
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = blockIdx.x / p.slices, s = blockIdx.x - m * p.slices;
    const int j0 = s * kU;

    if (warp == 4 && lane == 0) {
        tma_prefetch_desc(&tmH);
        tma_prefetch_desc(&tmW);
        mbar_init(wfull, 1);
        for (int i = 0; i < kAStages; ++i) {
            mbar_init(&afull[i], 1);
            mbar_init(&aempty[i], 4);  // one arrival per gate warp
        }
        fence_barrier_init();
    }
    if (threadIdx.x < kN) {
        const int g = threadIdx.x / kU, u = threadIdx.x - g * kU;
        sBias[threadIdx.x] = (j0 + u < p.Hd) ? p.bhh[g * p.Hd + j0 + u] : 0.f;
    }
    __syncthreads();

    if (warp == 4) {
        // ===================== TMA producer: the weight slice once, then h_{t-1} tiles step by step =====================
        if (elect_one()) {
            mbar_arrive_expect_tx(wfull, static_cast<uint32_t>(p.k_chunks * kWChunk));
            for (int c = 0; c < p.k_chunks; ++c)
                for (int g = 0; g < 3; ++g)  // rows beyond 3*Hd (last slice, gate n) are zero filled; rows of a neighbouring gate are finite and unused
                    tma_load_2d(sW + c * kWChunk + g * (kU * 128), &tmW, wfull, c * 64, g * p.Hd + j0);
        }
        __syncwarp();
        int st = 0;
        uint32_t ph = 0;
        for (int t = 0; t < p.S; ++t) {
            if (t > 0) {  // every slice of this row tile has published h_t
                if (lane == 0) {
                    const unsigned int want = static_cast<unsigned int>(t) * static_cast<unsigned int>(p.slices);
                    const uint64_t t0 = globaltimer_ns();
                    uint32_t spins = 0;
                    while (ld_acquire(p.bar + m) < want) {
                        __nanosleep(40);
                        if ((++spins & 0xfff) == 0 && globaltimer_ns() - t0 > 4000000000ull) f_timeout(401, static_cast<uint32_t>(t));
                    }
                    asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy writes of the other CTAs -> this CTA's TMA reads
                }
                __syncwarp();
            }
            for (int c = 0; c < p.k_chunks; ++c) {
                f_wait(&aempty[st], ph ^ 1u, 402);
                if (elect_one()) {
                    mbar_arrive_expect_tx(&afull[st], kAStage);
                    tma_load_2d(sA + st * kAStage, &tmH, &afull[st], c * 64, t * p.B + m * 128);
                }
                __syncwarp();
                if (++st == kAStages) { st = 0; ph ^= 1u; }
            }
        }
    } else {
        // ===================== gate warps: wgmma, then the gates in the accumulator fragment layout =====================
        // Fragment of m64n96 block bb: acc[bb][4j + 2e + i] = row 64bb + 16 * warp + lane / 4 + 8e, column 8j + 2 * (lane % 4) + i.
        // Gate g of unit u is column 32g + u, so the r, z and n pre-activations of (row, u) sit in the same thread:
        // j = jj (r), jj + 4 (z), jj + 8 (n) with u = 8jj + 2 * (lane % 4) + i.  Each thread owns 4 rows x 8 units.
        const uint32_t a_s = smem_u32(sA), w_s = smem_u32(sW);
        const int nvalid = min(kU, p.Hd - j0);  // units of this slice that exist (multiple of 4)
        const int uq = 2 * (lane & 3);
        int brow[2][2];
        bool valid[2][2];
        long long L[2][2];
        float h[2][2][4][2];
#pragma unroll
        for (int bb = 0; bb < 2; ++bb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                brow[bb][e] = m * 128 + 64 * bb + 16 * warp + (lane >> 2) + 8 * e;
                valid[bb][e] = brow[bb][e] < p.B;
                L[bb][e] = valid[bb][e] ? p.len[brow[bb][e]] : 1;
                if (L[bb][e] < 1) L[bb][e] = 1;  // reference clamps 0 -> 1 (user_encoder.py:27)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int u = 8 * jj + uq;
                    float2 v = make_float2(0.f, 0.f);
                    if (valid[bb][e] && u < nvalid) v = *reinterpret_cast<const float2*>(p.h0 + static_cast<size_t>(brow[bb][e]) * p.Hd + j0 + u);
                    h[bb][e][jj][0] = v.x;
                    h[bb][e][jj][1] = v.y;
                }
            }
        // the first wgmma reads the resident W_hh slice: its TMA loads, issued before the first A stage, may land after it
        f_wait(wfull, 0, 403);
        int st = 0;
        uint32_t ph = 0;
        for (int t = 0; t < p.S; ++t) {
            float acc[2][kN / 2];
            for (int c = 0; c < p.k_chunks; ++c) {
                f_wait(&afull[st], ph, 405);
                const uint64_t db = make_sw128_desc(w_s + c * kWChunk, 16, 1024);
#pragma unroll
                for (int bb = 0; bb < 2; ++bb)
#pragma unroll
                    for (int i = 0; i < kN / 2; ++i) wgmma_reg_fence(acc[bb][i]);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)  // columns past Hd are zero filled by TMA in both operands
#pragma unroll
                    for (int bb = 0; bb < 2; ++bb)
                        Wgmma<kN, 0, 0>::mma(acc[bb], make_sw128_desc(a_s + st * kAStage + bb * 8192, 16, 1024) + 2 * k, db + 2 * k,
                                             (c | k) ? 1 : 0);
                wgmma_commit();
                wgmma_wait<0>();
#pragma unroll
                for (int bb = 0; bb < 2; ++bb)
#pragma unroll
                    for (int i = 0; i < kN / 2; ++i) wgmma_reg_fence(acc[bb][i]);
                __syncwarp();
                if (lane == 0) mbar_arrive(&aempty[st]);
                if (++st == kAStages) { st = 0; ph ^= 1u; }
            }
#pragma unroll
            for (int bb = 0; bb < 2; ++bb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int b = valid[bb][e] ? brow[bb][e] : 0;
                    const float* girow = p.gi + (static_cast<size_t>(b) * p.S + t) * p.ldg + j0;
                    float* ghrow = p.gh + (static_cast<size_t>(t) * p.B + b) * p.ldg + j0;
                    float* hsrow = p.hs + (static_cast<size_t>(t + 1) * p.B + b) * p.Hd + j0;
                    __nv_bfloat16* hbrow = p.hb + (static_cast<size_t>(t + 1) * p.B + b) * p.ldh + j0;
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int u = 8 * jj + uq;
                        if (u >= nvalid) continue;
                        float x[3][2], gv[3][2];
#pragma unroll
                        for (int g = 0; g < 3; ++g) {
                            const float2 bv = *reinterpret_cast<const float2*>(sBias + g * kU + u);
                            x[g][0] = acc[bb][4 * (jj + 4 * g) + 2 * e] + bv.x;
                            x[g][1] = acc[bb][4 * (jj + 4 * g) + 2 * e + 1] + bv.y;
                            const float2 gg = __ldg(reinterpret_cast<const float2*>(girow + g * p.Hd + u));
                            gv[g][0] = gg.x;
                            gv[g][1] = gg.y;
                        }
                        if (valid[bb][e]) {
#pragma unroll
                            for (int g = 0; g < 3; ++g) *reinterpret_cast<float2*>(ghrow + g * p.Hd + u) = make_float2(x[g][0], x[g][1]);
                        }
                        if (t < L[bb][e]) {
#pragma unroll
                            for (int i = 0; i < 2; ++i) {
                                const float rg = fast_sigmoid(gv[0][i] + x[0][i]);
                                const float zg = fast_sigmoid(gv[1][i] + x[1][i]);
                                const float n = fast_tanh(gv[2][i] + rg * x[2][i]);
                                h[bb][e][jj][i] = (1.f - zg) * n + zg * h[bb][e][jj][i];
                            }
                        }
                        if (valid[bb][e]) {
                            *reinterpret_cast<float2*>(hsrow + u) = make_float2(h[bb][e][jj][0], h[bb][e][jj][1]);
                            *reinterpret_cast<uint32_t*>(hbrow + u) = pack_bf16x2(h[bb][e][jj][0], h[bb][e][jj][1]);
                        }
                    }
                    // the slice that ends at Hd also owns the ones column and the zero pad of the bf16 rows
                    if (valid[bb][e] && (lane & 3) == 0 && (nvalid < kU || j0 + kU == p.Hd)) {
                        for (int c = p.Hd; c < p.ldh; ++c)
                            p.hb[(static_cast<size_t>(t + 1) * p.B + b) * p.ldh + c] = __float2bfloat16_rn(c == p.Hd ? 1.0f : 0.f);
                    }
                }
            if (t + 1 < p.S) {
                __threadfence();                                   // this thread's h_{t+1} rows are visible GPU-wide ...
                asm volatile("bar.sync 1, 128;" ::: "memory");     // ... for all four gate warps ...
                if (threadIdx.x == 0) red_release(p.bar + m);      // ... before the slice counts as arrived
            }
        }
#pragma unroll
        for (int bb = 0; bb < 2; ++bb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (!valid[bb][e]) continue;
                float* o = p.out + static_cast<size_t>(brow[bb][e]) * p.Hd + j0;
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int u = 8 * jj + uq;
                    if (u < nvalid) *reinterpret_cast<float2*>(o + u) = make_float2(h[bb][e][jj][0], h[bb][e][jj][1]);
                }
            }
    }
}

}  // namespace gru

// 1 if the persistent recurrence covers this shape on this device (else the caller runs the per-step sequence)
// dynamic shared memory of one CTA: alignment slack + resident weight slice + A ring + barriers / bias
static size_t gru_smem_bytes(int Hd) {
    return 1024 + static_cast<size_t>(ceil_div(Hd, 64)) * gru::kWChunk + gru::kAStages * gru::kAStage + 1024;
}

int gru_persistent_supported(int B, int Hd) {
    using namespace gru;
    if (B < 1 || Hd < 32 || Hd % 4 != 0 || gru_smem_bytes(Hd) > 232448) return 0;
    const int row_tiles = ceil_div(B, 128), slices = ceil_div(Hd, kU);
    return row_tiles * slices <= num_sms() ? 1 : 0;
}

int gru_fwd_persistent(int B, int S, int Hd, int ldh, int ldg, const float* gi, const void* whh, const float* bhh, const float* h0,
                       const long long* len, float* gh, float* hs, void* hb, float* out, cudaStream_t stream) {
    using namespace gru;
    NR_REQUIRE(gru_persistent_supported(B, Hd), "gru_fwd_persistent: unsupported shape B=%d Hd=%d", B, Hd);
    NR_REQUIRE(ldh % 8 == 0 && ldh >= Hd + 1 && ldg % 4 == 0 && ldg >= 3 * Hd, "gru_fwd_persistent: pitches ldh=%d ldg=%d", ldh, ldg);
    Params p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.S = S; p.Hd = Hd; p.ldh = ldh; p.ldg = ldg;
    p.slices = ceil_div(Hd, kU);
    p.k_chunks = ceil_div(Hd, 64);
    p.gi = gi; p.bhh = bhh; p.h0 = h0; p.len = len; p.gh = gh; p.hs = hs;
    p.hb = static_cast<__nv_bfloat16*>(hb);
    p.out = out;
    const int row_tiles = ceil_div(B, 128);
    unsigned int* bar = nullptr;
    NR_CHECK_CUDA(cudaMallocAsync(&bar, sizeof(unsigned int) * row_tiles, stream));
    NR_CHECK_CUDA(cudaMemsetAsync(bar, 0, sizeof(unsigned int) * row_tiles, stream));
    p.bar = bar;
    CUtensorMap tmH, tmW;
    NR_PROPAGATE(make_tmap_bf16_2d(&tmH, hb, static_cast<int64_t>(S + 1) * B, Hd, ldh, 64, 128));
    NR_PROPAGATE(make_tmap_bf16_2d(&tmW, whh, 3 * static_cast<int64_t>(Hd), Hd, ldh, 64, kU));
    const size_t smem = gru_smem_bytes(Hd);
    NR_REQUIRE(smem <= 232448, "gru_fwd_persistent: %zu bytes of shared memory", smem);
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(gru_fwd_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
        attr_set = true;
    }
    ProfScope ps("gru_fwd_persistent", B, S, Hd, stream);
    void* args[] = {&tmH, &tmW, &p};
    NR_CHECK_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(gru_fwd_persistent_kernel), dim3(row_tiles * p.slices), dim3(kThreads),
                                              args, smem, stream));
    ++g_launches;
    NR_CHECK_CUDA(cudaFreeAsync(bar, stream));
    return 0;
}

}  // namespace nr
