// extern "C" surface, part 2: the title/abstract CNN encoder shared by NAML / LSTUR / TANR, the category
// "element" encoder of NAML, fp32 embedding lookups, a generic Linear and the ReLU-backward helper.
#include <cstring>

#include "../../include/newsrec_b200.h"
#include "nr_common.cuh"
#include "nr_ops.h"

using namespace nr;

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }
static const RowMapCfg kIdentity = {0, 0, 0, 0, 0};
static const DropoutCfg kNoDrop = {0.f, 0};
static inline long long align256(long long x) { return (x + 255) & ~255ll; }
static inline int ru8(int x) { return (x + 7) & ~7; }
static inline int ru16(int x) { return (x + 15) & ~15; }

// Every shape limit of the kernels the encoder chains is checked here, before the first launch: T <= kGemmTileRows because
// a pooling tile holds whole segments (gemm_additive_pool), F % 4 == 0 for the float4 dOut rows of pool_dscore.
static int check_cnn_shape(long long n_seq, int T, int d, int F, int q, int ldx, int ldf) {
    NR_REQUIRE(n_seq >= 0 && T >= 1 && T <= kGemmTileRows && d >= 8 && F >= 8 && q >= 1 && q <= 256,
               "cnn encoder: bad shape n_seq=%lld T=%d (at most %d) d=%d F=%d q=%d", n_seq, T, kGemmTileRows, d, F, q);
    NR_REQUIRE(ldx == ru8(d + 1) && ldf == ru8(F + 1), "cnn encoder: pitches must be round_up(width+1, 8) (ldx=%d ldf=%d)", ldx, ldf);
    NR_REQUIRE(d % 4 == 0 && F % 4 == 0, "cnn encoder: d and F must be multiples of 4 (d=%d F=%d)", d, F);
    NR_REQUIRE(n_seq * (T + 2) < (1ll << 31), "cnn encoder: too many rows");
    return 0;
}

extern "C" {

// ---- reference: TextEncoder / title_CNN + title_attention -------------------------------------------
//   NAML  src/model/NAML/news_encoder.py:21-37 ; LSTUR src/model/LSTUR/news_encoder.py:56-72 ;
//   TANR  src/model/TANR/news_encoder.py:40-52 :  embedding -> dropout -> Conv2d(1,F,(3,d),pad (1,0)) -> ReLU
//   -> dropout -> additive pooling
int nr_cnn_encoder_fwd(const nr_cnn_encoder_fwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_cnn_encoder_fwd: null args");
    NR_PROPAGATE(check_cnn_shape(a->n_seq, a->T, a->d, a->F, a->q, a->ldx, a->ldf));
    NR_REQUIRE(a->ids && a->table_bf16 && a->wconv_bf16 && a->bconv && a->wa_bf16 && a->ba && a->qv && a->Xp_bf16 && a->Y_bf16 &&
                   a->w && a->out && a->bad_id_flag, "nr_cnn_encoder_fwd: null operand");
    NR_REQUIRE(a->p_drop >= 0.f && a->p_drop < 1.f, "nr_cnn_encoder_fwd: dropout p=%f", a->p_drop);
    if (a->n_seq == 0) return 0;
    const cudaStream_t st = S(stream);
    const int T = a->T, Tp = T + 2;
    const long long n_tok = a->n_seq * T;
    const int Mp = static_cast<int>(a->n_seq * Tp);
    prof_context("cnn.fwd");
    NR_PROPAGATE(gather_rows(a->ids, n_tok, T, a->table_bf16, a->V, a->d, a->ldx, a->Xp_bf16, a->ldx, 1,
                             DropoutCfg{a->p_drop, a->seed}, a->bad_id_flag, st));
    const RowMapCfg to_compact = {Tp, 1, T, T, 0};
    NR_PROPAGATE(gemm_store(a->Xp_bf16, Mp, a->ldx, a->wconv_bf16, a->F, a->ldx, a->d, 3, a->F, kGemmTileRows, a->bconv, 1,
                            a->Y_bf16, a->ldf, 1, to_compact, 0, DropoutCfg{a->p_drop, a->seed ^ 0x5bd1e995u}, a->F, a->ldf, st,
                            a->Y_lo_bf16, a->ldf, 0));
    NR_PROPAGATE(gemm_additive_pool(a->Y_bf16, static_cast<int>(n_tok), a->ldf, a->F, a->wa_bf16, a->q, a->ldf, a->ba, a->qv, T,
                                    a->out, a->F, a->w, st, a->Y_lo_bf16));
    return 0;
}

long long nr_cnn_encoder_bwd_workspace(long long n_seq, int T, int F, int q) {
    const long long rows = n_seq * T, rows_p = n_seq * (T + 2);
    return align256(rows * 4) + align256(rows * ru16(q) * 2) + align256(rows_p * ru8(F + 1) * 2) + 256;
}

int nr_cnn_encoder_bwd(const nr_cnn_encoder_bwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_cnn_encoder_bwd: null args");
    NR_PROPAGATE(check_cnn_shape(a->n_seq, a->T, a->d, a->F, a->q, a->ldx, a->ldf));
    NR_REQUIRE(a->ldq == ru16(a->q), "nr_cnn_encoder_bwd: ldq=%d (must be round_up(q, 16))", a->ldq);
    NR_REQUIRE(a->ids && a->wconvT_bf16 && a->wa_bf16 && a->waT_bf16 && a->ba && a->qv && a->Xp_bf16 && a->Y_bf16 && a->w &&
                   a->dout && a->dWconv_ext && a->dWa_ext && a->dqv && a->demb && a->workspace, "nr_cnn_encoder_bwd: null operand");
    NR_REQUIRE(a->workspace_bytes >= nr_cnn_encoder_bwd_workspace(a->n_seq, a->T, a->F, a->q), "nr_cnn_encoder_bwd: workspace too small");
    if (a->n_seq == 0) return 0;
    const cudaStream_t st = S(stream);
    const int T = a->T, Tp = T + 2;
    const long long rows = a->n_seq * T;
    const int M = static_cast<int>(rows), Mp = static_cast<int>(a->n_seq * Tp);
    char* ws = static_cast<char*>(a->workspace);
    float* dscore = reinterpret_cast<float*>(ws);
    ws += align256(rows * 4);
    void* dpre = ws;
    ws += align256(rows * a->ldq * 2);
    void* dYp = ws;
    prof_context("cnn.bwd");
    // additive pooling backward; the ReLU / dropout of the conv output are folded into the dY epilogue, which
    // also re-maps the rows into the zero-padded layout the shifted (tap) loads below need
    NR_PROPAGATE(pool_dscore(a->Y_bf16, a->ldf, a->F, a->n_seq, T, a->w, a->dout, a->F, dscore, st));
    NR_PROPAGATE(gemm_additive_dpre(a->Y_bf16, M, a->ldf, a->F, a->wa_bf16, a->q, a->ldf, a->ba, a->qv, dscore, dpre, a->ldq,
                                    a->dqv, st));
    const RowMapCfg to_padded = {T, 0, T, Tp, 1};
    NR_PROPAGATE(gemm_pool_dinput(dpre, M, a->ldq, a->q, a->waT_bf16, a->F, a->ldq, a->w, a->dout, a->F, T, dYp, a->ldf, to_padded, 1,
                                  DropoutCfg{a->p_drop, a->seed ^ 0x5bd1e995u}, a->Y_bf16, a->ldf, st));
    NR_PROPAGATE(gemm_tn_accumulate(dpre, M, a->q, a->ldq, a->Y_bf16, M, a->F + 1, a->ldf, 0, a->F + 1, 0, a->dWa_ext, a->ldf, st));
    // conv weight gradient, one tap at a time: dW_s = dY^T . X[rows + (s-1)]; the ones column of X makes column d
    // of the centre tap the bias gradient
    for (int s = 0; s < 3; ++s)
        NR_PROPAGATE(gemm_tn_accumulate(dYp, Mp, a->F, a->ldf, a->Xp_bf16, Mp, a->d + 1, a->ldx, 0, a->d + 1, s - 1,
                                        a->dWconv_ext + static_cast<size_t>(s) * a->F * a->ldx, a->ldx, st));
    // embedding gradient: dX[r] = sum_s' W_(2-s')^T dY[r + s' - 1], scattered to the token ids
    const RowMapCfg to_compact = {Tp, 1, T, T, 0};
    NR_PROPAGATE(gemm_scatter_emb(dYp, Mp, a->ldf, a->wconvT_bf16, a->d, a->ldf, a->F, 3, a->d, kGemmTileRows, a->ids, a->demb,
                                  a->V, a->d, to_compact, DropoutCfg{a->p_drop, a->seed}, a->ldx, st));
    return 0;
}

// ---- generic Linear on dense fp32 rows (topic predictor, element encoder, GRU projections) -------------
int nr_linear_rows_fwd(const float* x, long long n, int K, long long s_row, long long s_col, void* X_bf16, int ldx,
                       const void* W_bf16, int N, int ldw, const float* bias, int relu, float* out, int ld_out, void* stream) {
    NR_REQUIRE(x && X_bf16 && W_bf16 && out && n >= 0 && n < (1ll << 31) && ldx == ru8(K + 1) && ld_out % 4 == 0,
               "nr_linear_rows_fwd: n=%lld K=%d ldx=%d ld_out=%d", n, K, ldx, ld_out);
    if (n == 0) return 0;
    prof_context("linear.fwd");
    NR_PROPAGATE(rows_to_bf16(x, n, 1, K, s_row, 0, s_col, X_bf16, ldx, S(stream)));
    return gemm_store(X_bf16, static_cast<int>(n), ldx, W_bf16, N, ldw, K, 1, 0, kGemmTileRows, bias, relu, out, ld_out, 0, kIdentity, 0, kNoDrop,
                      -1, 0, S(stream));
}

// dy (fp32 [n][N], optionally masked by relu_out > 0) -> dY bf16 ; dW_ext[N][ldx] += dY^T . [X | 1] ; dx = dY . W
int nr_linear_rows_bwd(const float* dy, const float* relu_out, long long n, int N, int ld_dy, void* dY_bf16, int ldn,
                       const void* X_bf16, int K, int ldx, const void* WT_bf16, int ldwT, float* dW_ext, float* dx, int ld_dx,
                       void* stream) {
    NR_REQUIRE(dy && dY_bf16 && X_bf16 && dW_ext && n >= 0 && n < (1ll << 31) && ldn == ru8(N + 1) && ldx == ru8(K + 1),
               "nr_linear_rows_bwd: n=%lld N=%d K=%d", n, N, K);
    if (n == 0) return 0;
    prof_context("linear.bwd");
    NR_PROPAGATE(relu_bwd_to_bf16(dy, relu_out, n, N, ld_dy, dY_bf16, ldn, S(stream)));
    for (int c0 = 0; c0 < K + 1; c0 += 512) {
        const int nb = (K + 1 - c0) < 512 ? (K + 1 - c0) : 512;
        NR_PROPAGATE(gemm_tn_accumulate(dY_bf16, static_cast<int>(n), N, ldn, X_bf16, static_cast<int>(n), K + 1, ldx, c0, nb, 0,
                                        dW_ext + c0, ldx, S(stream)));
    }
    if (dx != nullptr) {
        NR_REQUIRE(WT_bf16 && ld_dx % 4 == 0, "nr_linear_rows_bwd: transposed weight / dx pitch");
        NR_PROPAGATE(gemm_store(dY_bf16, static_cast<int>(n), ldn, WT_bf16, K, ldwT, N, 1, 0, kGemmTileRows, nullptr, 0, dx, ld_dx, 0, kIdentity, 0,
                                kNoDrop, -1, 0, S(stream)));
    }
    return 0;
}

// ---- fp32 embedding lookups (category / user tables: reference LSTUR/news_encoder.py:47-53, __init__.py:74) ----
int nr_embedding_f32_fwd(const long long* ids, long long n, const float* table, int V, int D, float* out, int* bad_id_flag,
                         void* stream) {
    NR_REQUIRE(ids && table && out && bad_id_flag && D >= 1, "nr_embedding_f32_fwd: null operand");
    return embedding_f32_fwd(ids, n, table, V, D, out, bad_id_flag, S(stream));
}
int nr_embedding_f32_bwd(const long long* ids, long long n, const float* dout, int V, int D, float* dtable, void* stream) {
    NR_REQUIRE(ids && dout && dtable && V >= 1, "nr_embedding_f32_bwd: null operand or V=%d", V);
    return embedding_f32_bwd(ids, n, dout, V, D, dtable, S(stream));
}

// ---- NAML ElementEncoder: relu(Linear(embedding(id)))  (reference NAML/news_encoder.py:40-47) ----------------
int nr_element_encoder_fwd(const long long* ids, long long n, const void* table_bf16, int V, int E, int lde, void* E_bf16,
                           const void* W_bf16, int F, const float* bias, float* out, int* bad_id_flag, void* stream) {
    NR_REQUIRE(ids && table_bf16 && E_bf16 && W_bf16 && bias && out && bad_id_flag && lde == ru8(E + 1) && F % 4 == 0 &&
                   n < (1ll << 31), "nr_element_encoder_fwd: bad argument (E=%d lde=%d F=%d)", E, lde, F);
    if (n == 0) return 0;
    prof_context("element.fwd");
    NR_PROPAGATE(gather_rows(ids, n, 1, table_bf16, V, E, lde, E_bf16, lde, 0, kNoDrop, bad_id_flag, S(stream)));
    return gemm_store(E_bf16, static_cast<int>(n), lde, W_bf16, F, lde, E, 1, 0, kGemmTileRows, bias, 1, out, F, 0, kIdentity, 0, kNoDrop, -1, 0,
                      S(stream));
}
int nr_element_encoder_bwd(const long long* ids, long long n, const float* dout, const float* out, int F, void* dY_bf16, int ldf,
                           const void* E_bf16, int E, int lde, const void* WT_bf16, float* dW_ext, float* dtable, int V, void* stream) {
    NR_REQUIRE(ids && dout && out && dY_bf16 && E_bf16 && WT_bf16 && dW_ext && dtable && ldf == ru8(F + 1) && lde == ru8(E + 1) &&
                   E % 4 == 0 && n < (1ll << 31) && V >= 1, "nr_element_encoder_bwd: bad argument");
    if (n == 0) return 0;
    prof_context("element.bwd");
    NR_PROPAGATE(relu_bwd_to_bf16(dout, out, n, F, F, dY_bf16, ldf, S(stream)));
    NR_PROPAGATE(gemm_tn_accumulate(dY_bf16, static_cast<int>(n), F, ldf, E_bf16, static_cast<int>(n), E + 1, lde, 0, E + 1, 0, dW_ext,
                                    lde, S(stream)));
    return gemm_scatter_emb(dY_bf16, static_cast<int>(n), ldf, WT_bf16, E, ldf, F, 1, 0, kGemmTileRows, ids, dtable, V, E, kIdentity, kNoDrop, lde,
                            S(stream));
}

}  // extern "C"
