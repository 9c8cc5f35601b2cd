// extern "C" surface, part 2: the title/abstract CNN encoder shared by NAML / LSTUR / TANR, the category
// "element" encoder of NAML, fp32 embedding lookups, a generic Linear and the ReLU-backward helper.
#include <algorithm>
#include <cstring>

#include "../../include/newsrec_b200.h"
#include "nr_common.cuh"
#include "nr_ops.h"

using namespace nr;

// Every shape limit of the kernels the encoder chains is checked here, before the first launch: T <= kGemmTileRows because
// a pooling tile holds whole segments (gemm_additive_pool), F % 4 == 0 for the float4 dOut rows of pool_dscore, a window
// of 1 to 4 taps (the conv GEMMs' limit; one zero pad row on each side of a segment covers all four) and at least one
// output position per segment.
static int check_cnn_shape(long long n_seq, int T, int d, int F, int q, int ldx, int ldf, int window) {
    NR_REQUIRE(window >= 1 && window <= 4, "cnn encoder: window=%d (1 .. 4)", window);
    NR_REQUIRE(n_seq >= 0 && T >= 1 && T <= kGemmTileRows && d >= 8 && F >= 8 && q >= 1 && q <= 256,
               "cnn encoder: bad shape n_seq=%lld T=%d (at most %d) d=%d F=%d q=%d", n_seq, T, kGemmTileRows, d, F, q);
    NR_REQUIRE(T >= window - 2 * ((window - 1) / 2), "cnn encoder: T=%d leaves no output position at window=%d", T, window);
    NR_REQUIRE(ldx == round_up(d + 1, 8) && ldf == round_up(F + 1, 8), "cnn encoder: pitches must be round_up(width+1, 8) (ldx=%d ldf=%d)", ldx, ldf);
    NR_REQUIRE(d % 4 == 0 && F % 4 == 0, "cnn encoder: d and F must be multiples of 4 (d=%d F=%d)", d, F);
    NR_REQUIRE(n_seq * (T + 2) < (1ll << 31), "cnn encoder: too many rows");
    return 0;
}

// The reference's Conv2d(1, F, (w, d), padding ((w - 1) / 2, 0)) over T tokens: pad rows p = (w - 1) / 2 on each side,
// L = T + 2p - w + 1 output positions (T at odd w, T - 1 at even w).  In the padded layout (token t at row t + 1 of a
// segment's T + 2 rows) output j reads rows j + 1 - p + s, s < w: the conv GEMM's taps with tap origin p.
struct CnnWindow {
    int w, p, L;
    CnnWindow(int window, int T) : w(window == 0 ? 3 : window), p((w - 1) / 2), L(T + 2 * p - w + 1) {}
};

extern "C" {

// ---- reference: TextEncoder / title_CNN + title_attention -------------------------------------------
//   NAML  src/model/NAML/news_encoder.py:21-37 ; LSTUR src/model/LSTUR/news_encoder.py:56-72 ;
//   TANR  src/model/TANR/news_encoder.py:40-52 :  embedding -> dropout -> Conv2d(1,F,(w,d),pad ((w-1)/2,0)) -> ReLU
//   -> dropout -> additive pooling
int nr_cnn_encoder_fwd(const nr_cnn_encoder_fwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_cnn_encoder_fwd: null args");
    const CnnWindow win(a->window, a->T);
    NR_PROPAGATE(check_cnn_shape(a->n_seq, a->T, a->d, a->F, a->q, a->ldx, a->ldf, win.w));
    NR_REQUIRE(a->ids && a->table_bf16 && a->wconv_bf16 && a->bconv && a->wa_bf16 && a->ba && a->qv && a->Xp_bf16 && a->Y_bf16 &&
                   a->w && a->out && a->bad_id_flag, "nr_cnn_encoder_fwd: null operand");
    NR_REQUIRE(a->p_drop >= 0.f && a->p_drop < 1.f, "nr_cnn_encoder_fwd: dropout p=%f", a->p_drop);
    if (a->n_seq == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    const int T = a->T, Tp = T + 2, L = win.L;
    const long long n_tok = a->n_seq * T;
    const int Mp = static_cast<int>(a->n_seq * Tp);
    prof_context("cnn.fwd");
    NR_PROPAGATE(gather_rows(a->ids, n_tok, T, a->table_bf16, a->V, a->d, a->ldx, a->Xp_bf16, a->ldx, 1,
                             DropoutCfg{a->p_drop, a->seed}, a->bad_id_flag, st));
    // padded row r of a segment is output j = r - 1 when j < L: the rows that read past the output positions are dropped
    const RowMapCfg to_compact = {Tp, 1, L, L, 0};
    NR_PROPAGATE(gemm_store({.A = a->Xp_bf16, .M = Mp, .lda = a->ldx, .W = a->wconv_bf16, .N = a->F, .ldw = a->ldx, .K = a->d, .taps = win.w,
                             .w_tap_rows = a->F, .tap_origin = win.p},
                            {.out = a->Y_bf16, .ld_out = a->ldf, .out_bf16 = 1, .relu = 1, .bias = a->bconv, .rm = to_compact,
                             .drop = context_dropout(a->p_drop, a->seed), .ones_col = a->F, .ones_zero_upto = a->ldf, .lo_out = a->Y_lo_bf16,
                             .ld_lo = a->ldf}, st));
    NR_PROPAGATE(gemm_additive_pool(a->Y_bf16, static_cast<int>(a->n_seq * L), a->ldf, a->F, a->wa_bf16, a->q, a->ldf, a->ba, a->qv, L,
                                    a->out, a->F, a->w, st, a->Y_lo_bf16));
    return 0;
}

struct CnnBwdWorkspace : WorkspaceLayout {
    float* dscore;
    __nv_bfloat16 *dpre, *dYp;  // dY in the padded layout (T + 2 rows per segment)
    CnnBwdWorkspace(void* base, long long n_seq, int T, int F, int q)
        : WorkspaceLayout{static_cast<char*>(base)}, dscore(take<float>(n_seq * T)), dpre(take<__nv_bfloat16>(n_seq * T * round_up(q, 16))),
          dYp(take<__nv_bfloat16>(n_seq * (T + 2) * round_up(F + 1, 8))) {}
};
long long nr_cnn_encoder_bwd_workspace(long long n_seq, int T, int F, int q) { return CnnBwdWorkspace(nullptr, n_seq, T, F, q).bytes(); }

int nr_cnn_encoder_bwd(const nr_cnn_encoder_bwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_cnn_encoder_bwd: null args");
    const CnnWindow win(a->window, a->T);
    NR_PROPAGATE(check_cnn_shape(a->n_seq, a->T, a->d, a->F, a->q, a->ldx, a->ldf, win.w));
    NR_REQUIRE(a->ldq == round_up(a->q, 16), "nr_cnn_encoder_bwd: ldq=%d (must be round_up(q, 16))", a->ldq);
    NR_REQUIRE(a->ids && a->wconvT_bf16 && a->wa_bf16 && a->waT_bf16 && a->ba && a->qv && a->Xp_bf16 && a->Y_bf16 && a->w &&
                   a->dout && a->dWconv_ext && a->dWa_ext && a->dqv && a->demb && a->workspace, "nr_cnn_encoder_bwd: null operand");
    const CnnBwdWorkspace ws(a->workspace, a->n_seq, a->T, a->F, a->q);  // L <= T: sized for every window
    NR_REQUIRE(a->workspace_bytes >= ws.bytes(), "nr_cnn_encoder_bwd: workspace too small");
    if (a->n_seq == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    const int T = a->T, Tp = T + 2, L = win.L;
    const int M = static_cast<int>(a->n_seq * L), Mp = static_cast<int>(a->n_seq * Tp);
    const RowMapCfg to_padded = {L, 0, L, Tp, 1}, to_compact = {Tp, 1, T, T, 0};
    prof_context("cnn.bwd");
    // additive pooling backward; the ReLU / dropout of the conv output are folded into the dY epilogue, which
    // also re-maps the rows into the zero-padded layout the shifted (tap) loads below need
    NR_PROPAGATE(pool_dscore(a->Y_bf16, a->ldf, a->F, a->n_seq, L, a->w, a->dout, a->F, ws.dscore, st));
    NR_PROPAGATE(gemm_additive_dpre(a->Y_bf16, M, a->ldf, a->F, a->wa_bf16, a->q, a->ldf, a->ba, a->qv, ws.dscore, ws.dpre, a->ldq,
                                    a->dqv, st));
    // dY sits at rows 1 .. L of a segment; the epilogue zeroes rows 0 and L + 1.  At an even window L = T - 1, and row T + 1
    // is zeroed here: every weight-gradient tap sums over all rows, and the transposed conv of w = 4 reads it
    if (L < T)
        NR_CHECK_CUDA(cudaMemset2DAsync(ws.dYp + static_cast<size_t>(T + 1) * a->ldf, sizeof(__nv_bfloat16) * Tp * a->ldf, 0,
                                        sizeof(__nv_bfloat16) * a->ldf, a->n_seq, st));
    NR_PROPAGATE(gemm_pool_dinput({.A = ws.dpre, .M = M, .lda = a->ldq, .W = a->waT_bf16, .N = a->F, .ldw = a->ldq, .K = a->q},
                                  {.w = a->w, .dout = a->dout, .ldo = a->F, .seg_len = L, .dx = ws.dYp, .ld_dx = a->ldf, .rm = to_padded,
                                   .zero_pad_rows = 1, .drop = context_dropout(a->p_drop, a->seed), .relu_src = a->Y_bf16, .relu_ld = a->ldf}, st));
    NR_PROPAGATE(gemm_weight_grad(ws.dpre, M, a->q, a->ldq, a->Y_bf16, a->F, a->ldf, a->dWa_ext, st));
    // conv weight gradient, one tap at a time: dW_s = dY^T . X[rows + s - p]; the ones column of X makes column d
    // of tap p (shift 0) the bias gradient
    for (int s = 0; s < win.w; ++s)
        NR_PROPAGATE(gemm_weight_grad(ws.dYp, Mp, a->F, a->ldf, a->Xp_bf16, a->d, a->ldx,
                                      a->dWconv_ext + static_cast<size_t>(s) * a->F * a->ldx, st, s - win.p));
    // embedding gradient, the transposed conv: dX[r] = sum_s' W_(w-1-s')^T dY[r + s' - (w - 1 - p)], w - 1 - p = w / 2 being the
    // GEMM's centred tap origin; scattered to the token ids
    NR_PROPAGATE(gemm_scatter_emb({.A = ws.dYp, .M = Mp, .lda = a->ldf, .W = a->wconvT_bf16, .N = a->d, .ldw = a->ldf, .K = a->F, .taps = win.w,
                                   .w_tap_rows = a->d},
                                  {.ids = a->ids, .demb = a->demb, .V = a->V, .rm = to_compact, .drop = {a->p_drop, a->seed}, .drop_ld = a->ldx},
                                  st));
    return 0;
}

}  // extern "C"

// ---- reference: DKN KCNN (src/model/DKN/KCNN.py:56-117, use_context=False) -------------------------------
// Every shape limit of the chain, checked before the first launch: taps <= 4 per conv GEMM, a pooling tile holds whole segments
// (T <= kGemmTileRows), d and de multiples of 4 for the embedding scatters, F even for the pooled rows.
template <class Args>
static int check_kcnn_shape(const Args* a) {
    NR_REQUIRE(a->n_win >= 1 && a->n_win <= 4, "kcnn encoder: %d windows (1 .. 4)", a->n_win);
    int max_x = 0;
    for (int w = 0; w < a->n_win; ++w) {
        NR_REQUIRE(a->win[w] >= 1 && a->win[w] <= 4, "kcnn encoder: window %d (1 .. 4)", a->win[w]);
        max_x = std::max(max_x, a->win[w]);
    }
    NR_REQUIRE(a->n_seq >= 0 && a->T >= max_x && a->T <= kGemmTileRows && a->d >= 8 && a->de >= 8 && a->F >= 8 && a->q >= 1 && a->q <= 256,
               "kcnn encoder: bad shape n_seq=%lld T=%d (max window %d .. %d) d=%d de=%d F=%d q=%d", a->n_seq, a->T, max_x, kGemmTileRows,
               a->d, a->de, a->F, a->q);
    NR_REQUIRE(a->d % 4 == 0 && a->de % 4 == 0 && a->F % 2 == 0, "kcnn encoder: d, de must be multiples of 4 and F even (d=%d de=%d F=%d)",
               a->d, a->de, a->F);
    NR_REQUIRE(a->ldx == 2 * round_up(a->d + 1, 8) && a->lde == round_up(a->de + 1, 8) && a->ldf == round_up(a->F + 1, 8) &&
                   a->ldo == a->n_win * round_up(a->F, 4),
               "kcnn encoder: pitches ldx=%d lde=%d ldf=%d ldo=%d", a->ldx, a->lde, a->ldf, a->ldo);
    NR_REQUIRE(a->n_seq * a->T < (1ll << 31), "kcnn encoder: too many rows");
    return 0;
}
static int kcnn_max_window(const int* win, int n_win) { return *std::max_element(win, win + n_win); }

extern "C" {

int nr_kcnn_encoder_fwd(const nr_kcnn_encoder_fwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_kcnn_encoder_fwd: null args");
    NR_PROPAGATE(check_kcnn_shape(a));
    NR_REQUIRE(a->word_ids && a->entity_ids && a->word_table_bf16 && a->entity_table_bf16 && a->mT_bf16 && a->mb && a->wconv_bf16 &&
                   a->bconv && a->wa_bf16 && a->ba && a->qv && a->X2_bf16 && a->E_bf16 && a->Y_bf16 && a->w && a->out && a->bad_id_flag,
               "nr_kcnn_encoder_fwd: null operand");
    if (a->n_seq == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    const int T = a->T, sec = a->ldx / 2, Fs = round_up(a->F, 4);
    const long long n_tok = a->n_seq * T;
    const int M = static_cast<int>(n_tok);
    auto* X2 = static_cast<__nv_bfloat16*>(a->X2_bf16);
    prof_context("kcnn.fwd");
    // the two channels side by side in X2: the word rows, then tanh(E M + b) written by the GEMM into the entity section
    NR_PROPAGATE(gather_rows(a->word_ids, n_tok, T, a->word_table_bf16, a->V, a->d, sec, X2, a->ldx, 0, DropoutCfg{}, a->bad_id_flag, st));
    NR_PROPAGATE(gather_rows(a->entity_ids, n_tok, T, a->entity_table_bf16, a->Ve, a->de, a->lde, a->E_bf16, a->lde, 0, DropoutCfg{},
                             a->bad_id_flag, st));
    NR_PROPAGATE(gemm_store({.A = a->E_bf16, .M = M, .lda = a->lde, .W = a->mT_bf16, .N = a->d, .ldw = a->lde, .K = a->de},
                            {.out = X2 + sec, .ld_out = a->ldx, .out_bf16 = 1, .tanh = 1, .bias = a->mb, .ones_col = a->d,
                             .ones_zero_upto = sec}, st));
    NR_CHECK_CUDA(cudaMemsetAsync(a->out, 0, sizeof(float) * a->n_seq * a->ldo, st));  // the section padding columns
    long long row0 = 0;
    int tap0 = 0;
    for (int w = 0; w < a->n_win; ++w) {
        const int x = a->win[w], L = T + 1 - x;
        auto* Y = static_cast<__nv_bfloat16*>(a->Y_bf16) + row0 * a->ldf;
        // position p of a title = sum_s W_s . X2[p + s]: the rows p > T - x read the next title and are dropped by the row map
        NR_PROPAGATE(gemm_store({.A = X2, .M = M, .lda = a->ldx, .W = static_cast<const __nv_bfloat16*>(a->wconv_bf16) +
                                     static_cast<size_t>(tap0) * a->F * a->ldx, .N = a->F, .ldw = a->ldx, .K = a->ldx, .taps = x,
                                 .w_tap_rows = a->F, .tap_origin = 0},
                                {.out = Y, .ld_out = a->ldf, .out_bf16 = 1, .relu = 1, .bias = a->bconv + w * a->F, .rm = {T, 0, L, L, 0},
                                 .ones_col = a->F, .ones_zero_upto = a->ldf}, st));
        NR_PROPAGATE(gemm_additive_pool(Y, static_cast<int>(a->n_seq * L), a->ldf, a->F, a->wa_bf16, a->q, a->ldf, a->ba, a->qv, L,
                                        a->out + w * Fs, a->ldo, a->w + row0, st));
        row0 += a->n_seq * L;
        tap0 += x;
    }
    return 0;
}

struct KcnnBwdWorkspace : WorkspaceLayout {
    float* dscore;
    __nv_bfloat16 *dpre, *dY, *dZ;  // dY: every window's section in the T-row layout; dZ: the entity channel before tanh
    KcnnBwdWorkspace(void* base, long long n_seq, int T, int d, int F, int q, int n_win)
        : WorkspaceLayout{static_cast<char*>(base)}, dscore(take<float>(n_seq * T)), dpre(take<__nv_bfloat16>(n_seq * T * round_up(q, 16))),
          dY(take<__nv_bfloat16>(n_seq * T * n_win * round_up(F + 1, 8))), dZ(take<__nv_bfloat16>(n_seq * T * round_up(d + 1, 8))) {}
};
long long nr_kcnn_encoder_bwd_workspace(long long n_seq, int T, int d, int F, int q, int n_win) {
    return KcnnBwdWorkspace(nullptr, n_seq, T, d, F, q, n_win).bytes();
}

int nr_kcnn_encoder_bwd(const nr_kcnn_encoder_bwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_kcnn_encoder_bwd: null args");
    NR_PROPAGATE(check_kcnn_shape(a));
    NR_REQUIRE(a->ldq == round_up(a->q, 16), "nr_kcnn_encoder_bwd: ldq=%d (must be round_up(q, 16))", a->ldq);
    NR_REQUIRE(a->word_ids && a->entity_ids && a->wT_word_bf16 && a->wT_entity_bf16 && a->m_bf16 && a->wa_bf16 && a->waT_bf16 && a->ba &&
                   a->qv && a->X2_bf16 && a->E_bf16 && a->Y_bf16 && a->w && a->dout && a->dWconv_ext && a->dM_ext && a->dWa_ext && a->dqv &&
                   a->dword && a->dentity && a->workspace, "nr_kcnn_encoder_bwd: null operand");
    const KcnnBwdWorkspace ws(a->workspace, a->n_seq, a->T, a->d, a->F, a->q, a->n_win);
    NR_REQUIRE(a->workspace_bytes >= ws.bytes(), "nr_kcnn_encoder_bwd: workspace too small");
    if (a->n_seq == 0) return 0;
    const cudaStream_t st = as_stream(stream);
    const int T = a->T, sec = a->ldx / 2, Fs = round_up(a->F, 4), ldy = a->n_win * a->ldf;
    const int M = static_cast<int>(a->n_seq * T);
    const auto* X2 = static_cast<const __nv_bfloat16*>(a->X2_bf16);
    prof_context("kcnn.bwd");
    // the rows past each window's last position and the section padding stay 0: the taps below read them
    NR_CHECK_CUDA(cudaMemsetAsync(ws.dY, 0, sizeof(__nv_bfloat16) * M * ldy, st));
    long long row0 = 0;
    int tap0 = 0;
    for (int w = 0; w < a->n_win; ++w) {
        const int x = a->win[w], L = T + 1 - x, Mw = static_cast<int>(a->n_seq * L);
        const auto* Y = static_cast<const __nv_bfloat16*>(a->Y_bf16) + row0 * a->ldf;
        const float* wr = a->w + row0;
        const float* dout = a->dout + w * Fs;
        __nv_bfloat16* dYw = ws.dY + w * a->ldf;
        // the padding columns of dout are 0, so the dot over Fs columns (Y's ones column included) is the dot over F
        NR_PROPAGATE(pool_dscore(Y, a->ldf, Fs, a->n_seq, L, wr, dout, a->ldo, ws.dscore, st));
        NR_PROPAGATE(gemm_additive_dpre(Y, Mw, a->ldf, a->F, a->wa_bf16, a->q, a->ldf, a->ba, a->qv, ws.dscore, ws.dpre, a->ldq, a->dqv, st));
        NR_PROPAGATE(gemm_pool_dinput({.A = ws.dpre, .M = Mw, .lda = a->ldq, .W = a->waT_bf16, .N = a->F, .ldw = a->ldq, .K = a->q},
                                      {.w = wr, .dout = dout, .ldo = a->ldo, .seg_len = L, .dx = dYw, .ld_dx = ldy, .rm = {L, 0, L, T, 0},
                                       .relu_src = Y, .relu_ld = a->ldf}, st));
        NR_PROPAGATE(gemm_weight_grad(ws.dpre, Mw, a->q, a->ldq, Y, a->F, a->ldf, a->dWa_ext, st));
        // dW_(w,s) = dY_w^T . X2[rows + s]; the entity section's ones column makes column sec + d the bias gradient
        for (int s = 0; s < x; ++s)
            NR_PROPAGATE(gemm_weight_grad(dYw, M, a->F, ldy, X2, sec + a->d, a->ldx,
                                          a->dWconv_ext + static_cast<size_t>(tap0 + s) * a->F * a->ldx, st, s));
        row0 += a->n_seq * L;
        tap0 += x;
    }
    // transposed conv of all windows at once: dX2[r] = sum_(w, s) W_(w,s)^T dY_w[r - s], tap s' = max x - 1 - s reads row r + s' - (max x - 1)
    const int taps = kcnn_max_window(a->win, a->n_win);
    const GemmOperands tconv{.A = ws.dY, .M = M, .lda = ldy, .W = nullptr, .N = a->d, .ldw = ldy, .K = ldy, .taps = taps, .w_tap_rows = a->d,
                             .tap_origin = taps - 1};
    GemmOperands g = tconv;
    g.W = a->wT_word_bf16;
    NR_PROPAGATE(gemm_scatter_emb(g, {.ids = a->word_ids, .demb = a->dword, .V = a->V}, st));
    g.W = a->wT_entity_bf16;
    NR_PROPAGATE(gemm_store(g, {.out = ws.dZ, .ld_out = sec, .out_bf16 = 1, .dtanh_src = X2 + sec, .dtanh_ld = a->ldx}, st));
    NR_PROPAGATE(gemm_weight_grad(ws.dZ, M, a->d, sec, a->E_bf16, a->de, a->lde, a->dM_ext, st));
    return gemm_scatter_emb({.A = ws.dZ, .M = M, .lda = sec, .W = a->m_bf16, .N = a->de, .ldw = sec, .K = a->d},
                            {.ids = a->entity_ids, .demb = a->dentity, .V = a->Ve}, st);
}

// ---- generic Linear on dense fp32 rows (topic predictor, element encoder, GRU projections) -------------
int nr_linear_rows_fwd(const float* x, long long n, int K, long long s_row, long long s_col, void* X_bf16, int ldx,
                       const void* W_bf16, int N, int ldw, const float* bias, int relu, float* out, int ld_out, void* stream) {
    NR_REQUIRE(x && X_bf16 && W_bf16 && out && n >= 0 && n < (1ll << 31) && ldx == round_up(K + 1, 8) && ld_out % 4 == 0,
               "nr_linear_rows_fwd: n=%lld K=%d ldx=%d ld_out=%d", n, K, ldx, ld_out);
    if (n == 0) return 0;
    prof_context("linear.fwd");
    NR_PROPAGATE(rows_to_bf16({.src = x, .n_rows = n, .D = K, .s_seq = s_row, .s_col = s_col, .width = ldx, .hi = X_bf16, .ld_hi = ldx,
                               .ones_col = 1},
                              kRowsToBf16, as_stream(stream)));
    return gemm_store({.A = X_bf16, .M = static_cast<int>(n), .lda = ldx, .W = W_bf16, .N = N, .ldw = ldw, .K = K},
                      {.out = out, .ld_out = ld_out, .relu = relu, .bias = bias}, as_stream(stream));
}

// dy (fp32 [n][N], optionally masked by relu_out > 0) -> dY bf16 ; dW_ext[N][ldx] += dY^T . [X | 1] ; dx = dY . W
int nr_linear_rows_bwd(const float* dy, const float* relu_out, long long n, int N, int ld_dy, void* dY_bf16, int ldn,
                       const void* X_bf16, int K, int ldx, const void* WT_bf16, int ldwT, float* dW_ext, float* dx, int ld_dx,
                       void* stream) {
    NR_REQUIRE(dy && dY_bf16 && X_bf16 && dW_ext && n >= 0 && n < (1ll << 31) && ldn == round_up(N + 1, 8) && ldx == round_up(K + 1, 8),
               "nr_linear_rows_bwd: n=%lld N=%d K=%d", n, N, K);
    if (n == 0) return 0;
    prof_context("linear.bwd");
    NR_PROPAGATE(relu_bwd_to_bf16(dy, relu_out, n, N, ld_dy, dY_bf16, ldn, as_stream(stream)));
    NR_PROPAGATE(gemm_weight_grad(dY_bf16, static_cast<int>(n), N, ldn, X_bf16, K, ldx, dW_ext, as_stream(stream)));
    if (dx != nullptr) {
        NR_REQUIRE(WT_bf16 && ld_dx % 4 == 0, "nr_linear_rows_bwd: transposed weight / dx pitch");
        NR_PROPAGATE(gemm_store({.A = dY_bf16, .M = static_cast<int>(n), .lda = ldn, .W = WT_bf16, .N = K, .ldw = ldwT, .K = N},
                                {.out = dx, .ld_out = ld_dx}, as_stream(stream)));
    }
    return 0;
}

// ---- fp32 embedding lookups (category / user tables: reference LSTUR/news_encoder.py:47-53, __init__.py:74) ----
int nr_embedding_f32_fwd(const long long* ids, long long n, const float* table, int V, int D, float* out, int* bad_id_flag,
                         void* stream) {
    NR_REQUIRE(ids && table && out && bad_id_flag && D >= 1, "nr_embedding_f32_fwd: null operand");
    return embedding_f32_fwd(ids, n, table, V, D, out, bad_id_flag, as_stream(stream));
}
int nr_embedding_f32_bwd(const long long* ids, long long n, const float* dout, int V, int D, float* dtable, void* stream) {
    NR_REQUIRE(ids && dout && dtable && V >= 1, "nr_embedding_f32_bwd: null operand or V=%d", V);
    return embedding_f32_bwd(ids, n, dout, V, D, dtable, as_stream(stream));
}

// ---- NAML ElementEncoder: relu(Linear(embedding(id)))  (reference NAML/news_encoder.py:40-47) ----------------
int nr_element_encoder_fwd(const long long* ids, long long n, const void* table_bf16, int V, int E, int lde, void* E_bf16,
                           const void* W_bf16, int F, const float* bias, float* out, int* bad_id_flag, void* stream) {
    NR_REQUIRE(ids && table_bf16 && E_bf16 && W_bf16 && bias && out && bad_id_flag && lde == round_up(E + 1, 8) && F % 4 == 0 &&
                   n < (1ll << 31), "nr_element_encoder_fwd: bad argument (E=%d lde=%d F=%d)", E, lde, F);
    if (n == 0) return 0;
    prof_context("element.fwd");
    NR_PROPAGATE(gather_rows(ids, n, 1, table_bf16, V, E, lde, E_bf16, lde, 0, DropoutCfg{}, bad_id_flag, as_stream(stream)));
    return gemm_store({.A = E_bf16, .M = static_cast<int>(n), .lda = lde, .W = W_bf16, .N = F, .ldw = lde, .K = E},
                      {.out = out, .ld_out = F, .relu = 1, .bias = bias}, as_stream(stream));
}
int nr_element_encoder_bwd(const long long* ids, long long n, const float* dout, const float* out, int F, void* dY_bf16, int ldf,
                           const void* E_bf16, int E, int lde, const void* WT_bf16, float* dW_ext, float* dtable, int V, void* stream) {
    NR_REQUIRE(ids && dout && out && dY_bf16 && E_bf16 && WT_bf16 && dW_ext && dtable && ldf == round_up(F + 1, 8) && lde == round_up(E + 1, 8) &&
                   E % 4 == 0 && n < (1ll << 31) && V >= 1, "nr_element_encoder_bwd: bad argument");
    if (n == 0) return 0;
    prof_context("element.bwd");
    NR_PROPAGATE(relu_bwd_to_bf16(dout, out, n, F, F, dY_bf16, ldf, as_stream(stream)));
    NR_PROPAGATE(gemm_weight_grad(dY_bf16, static_cast<int>(n), F, ldf, E_bf16, E, lde, dW_ext, as_stream(stream)));
    return gemm_scatter_emb({.A = dY_bf16, .M = static_cast<int>(n), .lda = ldf, .W = WT_bf16, .N = E, .ldw = ldf, .K = F},
                            {.ids = ids, .demb = dtable, .V = V, .drop_ld = lde}, as_stream(stream));
}

}  // extern "C"
