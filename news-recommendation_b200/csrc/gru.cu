// LSTUR user encoder: nn.GRU over the (left-padded) history, packed-sequence semantics, last hidden state.
// reference: src/model/LSTUR/user_encoder.py:16-45  (pack_padded_sequence(first len[b] steps) -> nn.GRU).
//
// The input projection is ONE wgmma GEMM over all (user, step) rows; the recurrent projection is a chain of
// S sequentially dependent [B x Hd] x [Hd x 3Hd] wgmma GEMMs (weight slices stay resident per launch, rows of
// one step are one or a few M tiles), each followed by a fused gate kernel.  Gate order r, z, n (torch):
//   r = sig(gi_r + gh_r), z = sig(gi_z + gh_z), n = tanh(gi_n + r * gh_n), h' = (1 - z) n + z h ;
// user b stops updating after len[b] steps.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "../../include/newsrec_b200.h"
#include "nr_common.cuh"
#include "nr_ops.h"

namespace nr {

// gi: fp32 [B*S][ldg] rows (b*S + t);  gh: fp32 [B][ldg];  h: fp32 [B][Hd] (in/out);
// hb_next: bf16 [B][ldh] operand of the next step (ones column at Hd)
__global__ void gru_gate_fwd_kernel(const float* __restrict__ gi, const float* __restrict__ gh, int ldg, float* __restrict__ h,
                                    __nv_bfloat16* __restrict__ hb_next, int ldh, const long long* __restrict__ len, int B, int S,
                                    int Hd, int t) {
    const long long total = static_cast<long long>(B) * ldh;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int b = static_cast<int>(i / ldh), j = static_cast<int>(i - static_cast<long long>(b) * ldh);
        if (j > Hd) { hb_next[i] = __float2bfloat16_rn(0.f); continue; }
        if (j == Hd) { hb_next[i] = __float2bfloat16_rn(1.0f); continue; }
        float hv = h[static_cast<size_t>(b) * Hd + j];
        const long long L = len[b] < 1 ? 1 : len[b];  // reference clamps 0 -> 1 (user_encoder.py:27)
        if (t < L) {
            const float* gir = gi + (static_cast<size_t>(b) * S + t) * ldg;
            const float* ghr = gh + static_cast<size_t>(b) * ldg;
            const float r = fast_sigmoid(gir[j] + ghr[j]);
            const float z = fast_sigmoid(gir[Hd + j] + ghr[Hd + j]);
            const float n = fast_tanh(gir[2 * Hd + j] + r * ghr[2 * Hd + j]);
            hv = (1.f - z) * n + z * hv;
            h[static_cast<size_t>(b) * Hd + j] = hv;
        }
        hb_next[i] = __float2bfloat16_rn(hv);
    }
}

// Backward of one step.  dh_in = dha + dhb (direct path + recurrent GEMM path of the step after).
// Writes dgi (bf16, rows b*S+t of [B*S][ldb]), dgh (bf16 [B][ldb]), dh_direct (fp32 [B][Hd]).
__global__ void gru_gate_bwd_kernel(const float* __restrict__ gi, const float* __restrict__ gh, int ldg, const float* __restrict__ hprev,
                                    const float* __restrict__ dha, int pa, const float* __restrict__ dhb, int pb,
                                    const long long* __restrict__ len, int B, int S, int Hd, int t, __nv_bfloat16* __restrict__ dgi,
                                    __nv_bfloat16* __restrict__ dgh, int ldb, float* __restrict__ dh_direct, int pd) {
    const long long total = static_cast<long long>(B) * Hd;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int b = static_cast<int>(i / Hd), j = static_cast<int>(i - static_cast<long long>(b) * Hd);
        const float dh = dha[static_cast<size_t>(b) * pa + j] + (dhb != nullptr ? dhb[static_cast<size_t>(b) * pb + j] : 0.f);
        const long long L = len[b] < 1 ? 1 : len[b];
        __nv_bfloat16* dgir = dgi + (static_cast<size_t>(b) * S + t) * ldb;
        __nv_bfloat16* dghr = dgh + static_cast<size_t>(b) * ldb;
        if (t >= L) {
            dgir[j] = dgir[Hd + j] = dgir[2 * Hd + j] = __float2bfloat16_rn(0.f);
            dghr[j] = dghr[Hd + j] = dghr[2 * Hd + j] = __float2bfloat16_rn(0.f);
            dh_direct[static_cast<size_t>(b) * pd + j] = dh;
            continue;
        }
        const float* gir = gi + (static_cast<size_t>(b) * S + t) * ldg;
        const float* ghr = gh + static_cast<size_t>(b) * ldg;
        const float r = fast_sigmoid(gir[j] + ghr[j]);
        const float z = fast_sigmoid(gir[Hd + j] + ghr[Hd + j]);
        const float ghn = ghr[2 * Hd + j];
        const float n = fast_tanh(gir[2 * Hd + j] + r * ghn);
        const float hp = hprev[i];
        const float dn = dh * (1.f - z);
        const float dz = dh * (hp - n);
        const float dpn = dn * (1.f - n * n);
        const float dpz = dz * z * (1.f - z);
        const float dpr = dpn * ghn * r * (1.f - r);
        dgir[j] = __float2bfloat16_rn(dpr);
        dgir[Hd + j] = __float2bfloat16_rn(dpz);
        dgir[2 * Hd + j] = __float2bfloat16_rn(dpn);
        dghr[j] = __float2bfloat16_rn(dpr);
        dghr[Hd + j] = __float2bfloat16_rn(dpz);
        dghr[2 * Hd + j] = __float2bfloat16_rn(dpn * r);
        dh_direct[static_cast<size_t>(b) * pd + j] = dh * z;
    }
}

__global__ void add2_kernel(const float* __restrict__ a, int pa, const float* __restrict__ b, int pb, float* __restrict__ out, int B, int Hd) {
    const long long n = static_cast<long long>(B) * Hd;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long r = i / Hd, j = i - r * Hd;
        out[i] = a[r * pa + j] + (b != nullptr ? b[r * pb + j] : 0.f);
    }
}
__global__ void zero_pad_cols_kernel(__nv_bfloat16* __restrict__ m, long long rows, int from, int ld) {
    const int w = ld - from;
    const long long total = rows * w;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long r = i / w;
        m[r * ld + from + (i - r * w)] = __float2bfloat16_rn(0.f);
    }
}

// Forward path switch: 1 = per-step sequence even where the persistent kernel applies.  Read lazily from NEWSREC_GRU_STEPWISE
// (set: 1) on the first forward unless nr_debug_set_gru_stepwise set it before; -1 = not decided yet.
static int g_gru_stepwise = -1;
static bool gru_stepwise() {
    if (g_gru_stepwise < 0) g_gru_stepwise = getenv("NEWSREC_GRU_STEPWISE") != nullptr ? 1 : 0;
    return g_gru_stepwise == 1;
}
void set_gru_stepwise(int on) { g_gru_stepwise = on ? 1 : 0; }

// the shape rules of nr_gru_fwd and nr_gru_bwd; the message names the rule a shape breaks
static int check_gru_shape(const char* fn, int B, int S, int D, int Hd) {
    NR_REQUIRE(B >= 0, "%s: B=%d is negative", fn, B);
    NR_REQUIRE(S >= 1, "%s: S=%d, at least one step is needed", fn, S);
    NR_REQUIRE(D >= 8 && D % 4 == 0, "%s: D=%d is not a multiple of 4 of at least 8", fn, D);
    NR_REQUIRE(Hd >= 8 && Hd % 2 == 0, "%s: Hd=%d is not an even number of at least 8", fn, Hd);
    return 0;
}

}  // namespace nr

using namespace nr;
static inline int blocks_for(long long n) { return static_cast<int>(std::min<long long>((n + 255) / 256, 148 * 8)); }

extern "C" {

// Saved-state sizes (elements): gi fp32 [B*S][ldg], gh fp32 [S][B][ldg], hs fp32 [S+1][B][Hd], hb bf16 [S+1][B][ldh],
// xb bf16 [B*S][ldd]   with ldg = round_up(3Hd, 4), ldh = round_up(Hd+1, 8), ldd = round_up(D+1, 8)
int nr_gru_fwd(const nr_gru_fwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_gru_fwd: null args");
    const int B = a->B, S = a->S, D = a->D, Hd = a->Hd;
    NR_PROPAGATE(check_gru_shape("nr_gru_fwd", B, S, D, Hd));
    NR_REQUIRE(a->x && a->len && a->h0 && a->wih_bf16 && a->whh_bf16 && a->bih && a->bhh && a->xb && a->gi && a->gh && a->hs && a->hb && a->out,
               "nr_gru_fwd: null operand");
    if (B == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    const int ldg = round_up(3 * Hd, 4), ldh = round_up(Hd + 1, 8), ldd = round_up(D + 1, 8);
    const long long BH = static_cast<long long>(B) * Hd;
    prof_context("gru.fwd");
    // gi = X Wih^T + bih over all (user, step) rows
    const Bf16Rows x_rows{.src = a->x, .n_rows = static_cast<long long>(B) * S, .T = S, .D = D, .s_seq = a->x_s_b, .s_tok = a->x_s_t,
                          .s_col = a->x_s_c, .width = ldd};
    Bf16Rows x_hi = x_rows;
    x_hi.hi = a->xb, x_hi.ld_hi = ldd, x_hi.ones_col = 1;
    NR_PROPAGATE(rows_to_bf16(x_hi, kRowsToBf16, st));
    NR_PROPAGATE(gemm_store({.A = a->xb, .M = B * S, .lda = ldd, .W = a->wih_bf16, .N = 3 * Hd, .ldw = ldd, .K = D},
                            {.out = a->gi, .ld_out = ldg, .bias = a->bih}, st));
    if (a->x_lo_bf16 != nullptr) {
        // accurate mode: the news vectors enter as a hi/lo bf16 pair, gi = x_hi . W_ih^T + b + x_lo . W_ih^T.  Two passes over the
        // SAME resident weights with fp32 accumulation into gi: a K-concatenated single pass doubles K, which shrinks the weight-
        // stationary slices to N = 80 and costs 0.86 ms instead of 2 x 0.23
        Bf16Rows x_lo = x_rows;  // no ones column: the bias belongs to the hi pass
        x_lo.lo = a->x_lo_bf16, x_lo.ld_lo = ldd;
        NR_PROPAGATE(rows_to_bf16(x_lo, kRowsToBf16Lo, st));
        NR_PROPAGATE(gemm_store({.A = a->x_lo_bf16, .M = B * S, .lda = ldd, .W = a->wih_bf16, .N = 3 * Hd, .ldw = ldd, .K = D},
                                {.out = a->gi, .ld_out = ldg, .accumulate = 1}, st));
    }
    // h_0
    NR_CHECK_CUDA(cudaMemcpyAsync(a->hs, a->h0, sizeof(float) * BH, cudaMemcpyDeviceToDevice, st));
    NR_PROPAGATE(rows_to_bf16({.src = a->h0, .n_rows = B, .D = Hd, .s_seq = Hd, .width = ldh, .hi = a->hb, .ld_hi = ldh, .ones_col = 1},
                              kRowsToBf16, st));
    if (!gru_stepwise() && gru_persistent_supported(B, Hd)) {
        // one cooperative launch for the whole recurrence (gru_persist.cu); same saved state as the per-step sequence below
        return gru_fwd_persistent(B, S, Hd, ldh, ldg, a->gi, a->whh_bf16, a->bhh, a->h0, a->len, a->gh, a->hs, a->hb, a->out, st);
    }
    for (int t = 0; t < S; ++t) {
        float* gh_t = a->gh + static_cast<size_t>(t) * B * ldg;
        const void* hb_t = static_cast<const __nv_bfloat16*>(a->hb) + static_cast<size_t>(t) * B * ldh;
        __nv_bfloat16* hb_n = static_cast<__nv_bfloat16*>(a->hb) + static_cast<size_t>(t + 1) * B * ldh;
        float* h_n = a->hs + static_cast<size_t>(t + 1) * BH;
        NR_PROPAGATE(gemm_store({.A = hb_t, .M = B, .lda = ldh, .W = a->whh_bf16, .N = 3 * Hd, .ldw = ldh, .K = Hd},
                                {.out = gh_t, .ld_out = ldg, .bias = a->bhh}, st));
        NR_CHECK_CUDA(cudaMemcpyAsync(h_n, a->hs + static_cast<size_t>(t) * BH, sizeof(float) * BH, cudaMemcpyDeviceToDevice, st));
        {
            ProfScope ps("gru_gate_fwd", B, Hd, t, st);
            gru_gate_fwd_kernel<<<blocks_for(static_cast<long long>(B) * ldh), 256, 0, st>>>(a->gi, gh_t, ldg, h_n, hb_n, ldh, a->len, B, S, Hd, t);
            ++g_launches;
        }
        NR_CHECK_CUDA(cudaGetLastError());
    }
    NR_CHECK_CUDA(cudaMemcpyAsync(a->out, a->hs + static_cast<size_t>(S) * BH, sizeof(float) * BH, cudaMemcpyDeviceToDevice, st));
    return 0;
}

int nr_gru_persistent_supported(int B, int Hd) { return gru_persistent_supported(B, Hd); }

// dgi bf16 [B*S][ldb] (rows b*S+t), dgh bf16 [S][B][ldb] with ldb = round_up(3Hd+1, 8); dh_direct / dh_rec fp32 [B][round_up(Hd, 4)]
struct GruBwdWorkspace : WorkspaceLayout {
    __nv_bfloat16 *dgi, *dgh;
    float *dh_direct, *dh_rec;
    GruBwdWorkspace(void* base, long long B, int S, int Hd)
        : WorkspaceLayout{static_cast<char*>(base)}, dgi(take<__nv_bfloat16>(B * S * round_up(3 * Hd + 1, 8))),
          dgh(take<__nv_bfloat16>(B * S * round_up(3 * Hd + 1, 8))), dh_direct(take<float>(B * round_up(Hd, 4))),
          dh_rec(take<float>(B * round_up(Hd, 4))) {}
};
long long nr_gru_bwd_workspace(int B, int S, int D, int Hd) { return GruBwdWorkspace(nullptr, B, S, Hd).bytes(); }

int nr_gru_bwd(const nr_gru_bwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_gru_bwd: null args");
    const int B = a->B, S = a->S, D = a->D, Hd = a->Hd;
    NR_PROPAGATE(check_gru_shape("nr_gru_bwd", B, S, D, Hd));
    NR_REQUIRE(a->len && a->wihT_bf16 && a->whhT_bf16 && a->xb && a->gi && a->gh && a->hs && a->hb && a->dout && a->dWih_ext && a->dWhh_ext &&
                   a->dx && a->dh0 && a->workspace, "nr_gru_bwd: null operand");
    const GruBwdWorkspace ws(a->workspace, B, S, Hd);
    NR_REQUIRE(a->workspace_bytes >= ws.bytes(), "nr_gru_bwd: workspace too small: %lld bytes, nr_gru_bwd_workspace gives %lld",
               a->workspace_bytes, ws.bytes());
    if (B == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    const int ldg = round_up(3 * Hd, 4), ldh = round_up(Hd + 1, 8), ldd = round_up(D + 1, 8), ldb = round_up(3 * Hd + 1, 8);
    const long long BH = static_cast<long long>(B) * Hd;
    const int P = round_up(Hd, 4);  // pitch of the internal dh buffers (fp32 vector stores of the GEMM epilogue)
    prof_context("gru.bwd");
    {   // pad columns [3Hd, ldb) of both gradient matrices are K-extent-masked by TMA but read by nothing else: keep them clean
        zero_pad_cols_kernel<<<blocks_for(static_cast<long long>(B) * S * (ldb - 3 * Hd)), 256, 0, st>>>(ws.dgi, static_cast<long long>(B) * S, 3 * Hd, ldb);
        zero_pad_cols_kernel<<<blocks_for(static_cast<long long>(B) * S * (ldb - 3 * Hd)), 256, 0, st>>>(ws.dgh, static_cast<long long>(B) * S, 3 * Hd, ldb);
        g_launches += 2;
    }
    const float* dha = a->dout;
    const float* dhb = nullptr;
    int pa = Hd;
    for (int t = S - 1; t >= 0; --t) {
        const float* gh_t = a->gh + static_cast<size_t>(t) * B * ldg;
        __nv_bfloat16* dgh_t = ws.dgh + static_cast<size_t>(t) * B * ldb;
        {
            ProfScope ps("gru_gate_bwd", B, Hd, t, st);
            gru_gate_bwd_kernel<<<blocks_for(BH), 256, 0, st>>>(a->gi, gh_t, ldg, a->hs + static_cast<size_t>(t) * BH, dha, pa, dhb, P, a->len, B, S,
                                                               Hd, t, ws.dgi, dgh_t, ldb, ws.dh_direct, P);
            ++g_launches;
        }
        NR_CHECK_CUDA(cudaGetLastError());
        // recurrent path: dh_{t-1} += dgh_t . Whh
        NR_PROPAGATE(gemm_store({.A = dgh_t, .M = B, .lda = ldb, .W = a->whhT_bf16, .N = Hd, .ldw = ldb, .K = 3 * Hd},
                                {.out = ws.dh_rec, .ld_out = P}, st));
        dha = ws.dh_direct;
        dhb = ws.dh_rec;
        pa = P;
    }
    add2_kernel<<<blocks_for(BH), 256, 0, st>>>(dha, pa, dhb, P, a->dh0, B, Hd);
    ++g_launches;
    // weight gradients over all (step, user) rows; the ones column of the saved operands yields the bias gradients
    NR_PROPAGATE(gemm_weight_grad(ws.dgh, B * S, 3 * Hd, ldb, a->hb, Hd, ldh, a->dWhh_ext, st));
    NR_PROPAGATE(gemm_weight_grad(ws.dgi, B * S, 3 * Hd, ldb, a->xb, D, ldd, a->dWih_ext, st));
    // input gradient
    NR_PROPAGATE(gemm_store({.A = ws.dgi, .M = B * S, .lda = ldb, .W = a->wihT_bf16, .N = D, .ldw = ldb, .K = 3 * Hd},
                            {.out = a->dx, .ld_out = D}, st));
    return 0;
}

}  // extern "C"
