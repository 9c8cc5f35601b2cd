// extern "C" surface declared in include/newsrec_b200.h: argument validation + kernel sequencing.
#include <cstring>
#include <utility>

#include "../../include/newsrec_b200.h"
#include "nr_common.cuh"
#include "nr_ops.h"

namespace nr {
const char* last_error();
int read_device_error(int* out4);
void set_debug_simt_gemm(int on);
int has_triage_backends();
void set_debug_gemm_timing(void* dev_buf, int slots);
void set_comm_reserved_sms(int n);
}  // namespace nr

using namespace nr;

extern "C" {

int nr_version(void) { return 1; }
const char* nr_last_error(void) { return last_error(); }
int nr_device_error(int out4[4]) { return read_device_error(out4); }
long long nr_launch_count(void) { return g_launches; }
int nr_num_sms(void) { return num_sms(); }
void nr_debug_set_simt_gemm(int on) { set_debug_simt_gemm(on); }
void nr_debug_set_gru_stepwise(int on) { set_gru_stepwise(on); }
int nr_debug_gemm_store(const nr_gemm_store_args* a, void* stream) {
    NR_REQUIRE(a && a->A && a->W && a->out, "nr_debug_gemm_store: null operand");
    const auto misaligned = [](const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; };
    NR_REQUIRE(!misaligned(a->out, 16) && !misaligned(a->lo_out, 16) && !misaligned(a->dtanh_src, 4),
               "nr_debug_gemm_store: out and lo_out need 16-byte, dtanh_src 4-byte aligned bases");
    return gemm_store({.A = a->A, .M = a->M, .lda = a->lda, .W = a->W, .N = a->N, .ldw = a->ldw, .K = a->K, .taps = a->taps,
                       .w_tap_rows = a->w_tap_rows, .tap_origin = a->tap_origin},
                      {.out = a->out, .ld_out = a->ld_out, .out_bf16 = a->out_bf16, .relu = a->relu, .tanh = a->tanh,
                       .dtanh_src = a->dtanh_src, .dtanh_ld = a->dtanh_ld, .bias = a->bias,
                       .rm = {a->rm_seg_in, a->rm_in_off, a->rm_seg_len, a->rm_seg_out, a->rm_out_off},
                       .drop = {a->p_drop, a->seed}, .ones_col = a->ones_col, .ones_zero_upto = a->ones_zero_upto, .lo_out = a->lo_out,
                       .ld_lo = a->ld_lo, .lo_col0 = a->lo_col0, .accumulate = a->accumulate, .rows_per_tile = a->rows_per_tile},
                      as_stream(stream));
}
int nr_debug_live_tokens(const long long* ids, long long n_seq, int T, int d, const void* table, int V, const void* X, int ldx,
                         const float* bqkv, unsigned* mask, unsigned char* pad, int* offset, int* index, int* tiles, void* Xc,
                         void* dqkv_c, void* stream) {
    NR_REQUIRE(ids && X && bqkv && mask && pad && offset && index && tiles && Xc && dqkv_c && n_seq >= 0 && d >= 2,
               "nr_debug_live_tokens: null operand or n_seq=%lld d=%d", n_seq, d);
    const cudaStream_t st = as_stream(stream);
    const int sec = (d + 7) & ~7, ld3 = (3 * sec + 15) & ~15;
    const long long bytes = live_tokens_bytes(n_seq, T, sec, ld3);
    char* buf = nullptr;
    NR_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&buf), bytes, st));
    LiveTokens lt;
    int rc = live_tokens(ids, n_seq, T, d, table, ldx, V, bqkv, sec, ld3, X, ldx, Xc, dqkv_c, buf, bytes, &lt, st);
    const size_t n = static_cast<size_t>(n_seq), M = n * T;
    const std::pair<void*, const void*> copies[] = {{mask, lt.mask}, {pad, lt.pad}, {offset, lt.offset}, {index, lt.index}, {tiles, lt.tiles}};
    const size_t sizes[] = {4 * n, n, 4 * (n + 1), 4 * M, 4 * (1 + (M + 63) / 64)};
    for (int i = 0; i < 5 && rc == 0 && n > 0; ++i)
        if (cudaMemcpyAsync(copies[i].first, copies[i].second, sizes[i], cudaMemcpyDeviceToDevice, st) != cudaSuccess) rc = -1;
    NR_CHECK_CUDA(cudaFreeAsync(buf, st));
    NR_REQUIRE(rc != -1, "nr_debug_live_tokens: copy-out failed");
    return rc;
}
int nr_has_triage_backends(void) { return has_triage_backends(); }
void nr_reserve_sms_for_comm(int n) { set_comm_reserved_sms(n); }
void nr_debug_set_gemm_timing(void* dev_buf, int slots) { set_debug_gemm_timing(dev_buf, slots); }
void nr_profile_enable(int on) { prof_enable(on); }
void nr_profile_context(const char* ctx) { prof_context(ctx ? ctx : ""); }
int nr_profile_report(char* buf, int cap) { return prof_report(buf, cap); }

// the zero-padded bf16 operand of an fp32 [R][C] matrix of pitch lds, or of its transpose
static Bf16Rows cast_pad_job(const float* src, int R, int C, int lds, void* dst, int ld, int transpose) {
    if (transpose) return {.src = src, .n_rows = C, .D = R, .s_seq = 1, .s_col = lds, .width = ld, .hi = dst, .ld_hi = ld};
    return {.src = src, .n_rows = R, .D = C, .s_seq = lds, .width = ld, .hi = dst, .ld_hi = ld};
}
int nr_cast_pad_bf16_many(int n, const float* const* src, const int* R, const int* C, const int* lds, void* const* dst, const int* ld,
                          const int* transpose, void* stream) {
    NR_REQUIRE(src && R && C && lds && dst && ld && transpose, "nr_cast_pad_bf16_many: null argument array");
    NR_REQUIRE(n >= 0 && n <= kBf16RowsJobs, "nr_cast_pad_bf16_many: %d matrices (at most %d per call)", n, kBf16RowsJobs);
    Bf16Rows jobs[kBf16RowsJobs];
    for (int i = 0; i < n; ++i) {
        NR_REQUIRE(R[i] >= 1 && C[i] >= 1, "nr_cast_pad_bf16_many: bad matrix %d", i);
        jobs[i] = cast_pad_job(src[i], R[i], C[i], lds[i], dst[i], ld[i], transpose[i]);
    }
    return rows_to_bf16(jobs, n, kCastPadMany, as_stream(stream));
}
int nr_cast_pad_bf16(const float* src, int R, int C, int lds, void* dst, int ld, int transpose, void* stream) {
    NR_REQUIRE(src && dst && R >= 0 && C >= 0 && ld % 8 == 0 && ld >= (transpose ? R : C),
               "nr_cast_pad_bf16: R=%d C=%d ld=%d transpose=%d", R, C, ld, transpose);
    return rows_to_bf16(cast_pad_job(src, R, C, lds, dst, ld, transpose), kCastPad, as_stream(stream));
}
int nr_rows_to_bf16(const float* src, long long n, int D, long long s_row, long long s_col, void* dst, int ld,
                    void* stream) {
    NR_REQUIRE(src && dst && n >= 0 && ld % 8 == 0, "nr_rows_to_bf16: n=%lld ld=%d", n, ld);
    return rows_to_bf16({.src = src, .n_rows = n, .D = D, .s_seq = s_row, .s_col = s_col, .width = ld, .hi = dst, .ld_hi = ld, .ones_col = 1},
                        kRowsToBf16, as_stream(stream));
}
int nr_rows_to_bf16_hilo(const float* src, long long n, int D, long long s_row, long long s_col, void* hi, void* lo, int ld,
                         void* stream) {
    NR_REQUIRE(src && hi && lo && n >= 0 && D >= 1 && ld % 8 == 0, "nr_rows_to_bf16_hilo: n=%lld D=%d ld=%d", n, D, ld);
    return rows_to_bf16({.src = src, .n_rows = n, .D = D, .s_seq = s_row, .s_col = s_col, .width = ld, .hi = hi, .ld_hi = ld, .ones_col = 1,
                         .lo = lo, .ld_lo = ld},
                        kRowsToBf16Planes, as_stream(stream));
}
int nr_gather_rows(const long long* ids, long long n_tok, int T, const void* table, int V, int D, int ld, void* X,
                   int padded, float p_drop, unsigned long long seed, int* bad_id_flag, void* stream) {
    NR_REQUIRE(ids && table && X && bad_id_flag && T >= 1 && n_tok % T == 0 && p_drop >= 0.f && p_drop < 1.f,
               "nr_gather_rows: n_tok=%lld T=%d p=%f", n_tok, T, p_drop);
    return gather_rows(ids, n_tok, T, table, V, D, ld, X, ld, padded, DropoutCfg{p_drop, seed}, bad_id_flag, as_stream(stream));
}
int nr_linear(const void* A, int M, int lda, const void* W, int N, int ldw, int K, int taps, int w_tap_rows,
              int rows_per_tile, const float* bias, int relu, void* out, int ld_out, int out_is_bf16, void* stream) {
    NR_REQUIRE(A && W && out && (taps == 1 || taps == 3), "nr_linear: null operand or taps=%d", taps);
    return gemm_store({.A = A, .M = M, .lda = lda, .W = W, .N = N, .ldw = ldw, .K = K, .taps = taps, .w_tap_rows = w_tap_rows},
                      {.out = out, .ld_out = ld_out, .out_bf16 = out_is_bf16, .relu = relu, .bias = bias, .rows_per_tile = rows_per_tile},
                      as_stream(stream));
}
int nr_gemm_tn(const void* A, int Kr, int Ma, int lda, const void* B, int b_rows, int b_cols, int ldb, int b_col0,
               int Nb, int b_row_shift, float* D, int ldd, void* stream) {
    NR_REQUIRE(A && B && D, "nr_gemm_tn: null operand");
    return gemm_tn_accumulate(A, Kr, Ma, lda, B, b_rows, b_cols, ldb, b_col0, Nb, b_row_shift, D, ldd, as_stream(stream));
}
int nr_mhsa_core_fwd(const void* qkv, int ld_qkv, int sec, long long n_seq, int T, int heads, int dk, void* ctx, int ld_ctx,
                     float p_drop, unsigned long long seed, void* stream) {
    NR_REQUIRE(qkv && ctx, "nr_mhsa_core_fwd: null operand");
    return mhsa_core_fwd(qkv, ld_qkv, sec, n_seq, T, heads, dk, ctx, ld_ctx, DropoutCfg{p_drop, seed}, as_stream(stream));
}
int nr_mhsa_core_bwd(const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int T, int heads,
                     int dk, void* dqkv, int ld_dqkv, void* stream) {
    NR_REQUIRE(qkv && dctx && dqkv, "nr_mhsa_core_bwd: null operand");
    return mhsa_core_bwd(qkv, ld_qkv, sec, dctx, ld_dctx, n_seq, T, heads, dk, dqkv, ld_dqkv, as_stream(stream));
}

// ---- AdditiveAttention ---------------------------------------------------------------------------
int nr_additive_attention_fwd(const void* X, long long n_seg, int seg_len, int D, int ldx, const void* Wa, int q, int ldw,
                              const float* ba, const float* qv, float* out, int ldo, float* w_out, void* stream) {
    NR_REQUIRE(X && Wa && ba && qv && out, "nr_additive_attention_fwd: null operand");
    NR_REQUIRE(n_seg * seg_len < (1ll << 31), "nr_additive_attention_fwd: too many rows");
    return gemm_additive_pool(X, static_cast<int>(n_seg * seg_len), ldx, D, Wa, q, ldw, ba, qv, seg_len, out, ldo, w_out,
                              as_stream(stream));
}
int nr_additive_attention_fwd_hilo(const void* X, const void* X_lo, long long n_seg, int seg_len, int D, int ldx, const void* Wa,
                                   int q, int ldw, const float* ba, const float* qv, float* out, int ldo, float* w_out, void* stream) {
    NR_REQUIRE(X && X_lo && Wa && ba && qv && out, "nr_additive_attention_fwd_hilo: null operand");
    NR_REQUIRE(n_seg * seg_len < (1ll << 31), "nr_additive_attention_fwd_hilo: too many rows");
    return gemm_additive_pool(X, static_cast<int>(n_seg * seg_len), ldx, D, Wa, q, ldw, ba, qv, seg_len, out, ldo, w_out,
                              as_stream(stream), X_lo);
}
struct AdditiveBwdWorkspace : WorkspaceLayout {
    float* dscore;
    __nv_bfloat16* dpre;  // [rows][round_up(q, 16)]
    AdditiveBwdWorkspace(void* base, long long rows, int q)
        : WorkspaceLayout{static_cast<char*>(base)}, dscore(take<float>(rows)), dpre(take<__nv_bfloat16>(rows * round_up(q, 16))) {}
};
long long nr_additive_attention_bwd_workspace(long long n_seg, int seg_len, int q) {
    return AdditiveBwdWorkspace(nullptr, n_seg * seg_len, q).bytes();
}
int nr_additive_attention_bwd(const void* X, long long n_seg, int seg_len, int D, int ldx, const void* Wa,
                              const void* WaT, int q, int ldw, int ldwT, const float* ba, const float* qv, const float* w,
                              const float* dout, int ldo, void* dX, int ld_dx, float* dWa_ext, float* dqv,
                              void* workspace, long long workspace_bytes, void* stream) {
    NR_REQUIRE(X && Wa && WaT && ba && qv && w && dout && dX && dWa_ext && dqv && workspace,
               "nr_additive_attention_bwd: null operand");
    // Every shape is checked before the first launch: the stages run in a row and dqv / dWa_ext accumulate, so a shape refused
    // by a later stage would return an error after an earlier one had changed them.  w comes from the forward: seg_len <= 64.
    NR_REQUIRE(n_seg >= 0 && seg_len >= 1 && seg_len <= 64 && q >= 1 && q <= 256 && D >= 4 && D % 4 == 0,
               "nr_additive_attention_bwd: bad shape n_seg=%lld seg_len=%d D=%d q=%d", n_seg, seg_len, D, q);
    NR_REQUIRE(ldx % 8 == 0 && ldx >= D + 1 && ldw % 8 == 0 && ldw >= D && ldwT % 8 == 0 && ldwT >= q && ldo % 4 == 0 && ldo >= D &&
                   ld_dx % 8 == 0 && ld_dx >= D,
               "nr_additive_attention_bwd: bad pitches ldx=%d ldw=%d ldwT=%d ldo=%d ld_dx=%d (D=%d q=%d)", ldx, ldw, ldwT, ldo, ld_dx, D, q);
    const auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };  // TMA bases, 16-byte dOut loads
    NR_REQUIRE(a16(X) && a16(Wa) && a16(WaT) && a16(dout) && a16(dX) && a16(workspace), "nr_additive_attention_bwd: operand not 16-byte aligned");
    const long long rows = n_seg * seg_len;
    NR_REQUIRE(rows < (1ll << 31), "nr_additive_attention_bwd: too many rows");
    const AdditiveBwdWorkspace ws(workspace, rows, q);
    NR_REQUIRE(workspace_bytes >= ws.bytes(), "nr_additive_attention_bwd: workspace too small");
    const int M = static_cast<int>(rows);
    const int ldq = round_up(q, 16);
    const GemmOperands dx_gemm{.A = ws.dpre, .M = M, .lda = ldq, .W = WaT, .N = D, .ldw = ldwT, .K = q};
    const PoolDInputCfg dx_cfg{.w = w, .dout = dout, .ldo = ldo, .seg_len = seg_len, .dx = dX, .ld_dx = ld_dx};
    NR_PROPAGATE(pool_dscore_check(ldx, D, seg_len, ldo));
    NR_PROPAGATE(additive_dpre_check(q, D, ldq));
    NR_PROPAGATE(pool_dinput_check(dx_gemm, dx_cfg));
    if (M == 0) return 0;
    NR_PROPAGATE(pool_dscore(X, ldx, D, n_seg, seg_len, w, dout, ldo, ws.dscore, as_stream(stream)));
    NR_PROPAGATE(gemm_additive_dpre(X, M, ldx, D, Wa, q, ldw, ba, qv, ws.dscore, ws.dpre, ldq, dqv, as_stream(stream)));
    NR_PROPAGATE(gemm_pool_dinput(dx_gemm, dx_cfg, as_stream(stream)));
    NR_PROPAGATE(gemm_weight_grad(ws.dpre, M, q, ldq, X, D, ldx, dWa_ext, as_stream(stream)));  // the ones column of X: d(bias)
    return 0;
}

int nr_dot_score_fwd(const float* cand, const float* user, int B, int C, int D, float* logits, void* stream) {
    NR_REQUIRE(cand && user && logits, "nr_dot_score_fwd: null operand");
    return dot_score_fwd(cand, user, B, C, D, logits, as_stream(stream));
}
int nr_dot_score_bwd(const float* cand, const float* user, const float* dlogits, int B, int C, int D, float* dcand,
                     float* duser, void* stream) {
    NR_REQUIRE(cand && user && dlogits && dcand && duser, "nr_dot_score_bwd: null operand");
    return dot_score_bwd(cand, user, dlogits, B, C, D, dcand, duser, as_stream(stream));
}


int nr_segment_dot(const float* news, long long n_news, int D, const long long* cand, long long n_cand, const long long* seg_offsets,
                   long long n_seg, const float* user, float* scores, int* bad_id_flag, void* stream) {
    NR_REQUIRE(news && cand && seg_offsets && user && scores && bad_id_flag && n_seg >= 1 && D >= 1 && n_cand >= 0,
               "nr_segment_dot: null operand or empty problem");
    return segment_dot(news, n_news, D, cand, n_cand, seg_offsets, n_seg, user, scores, bad_id_flag, as_stream(stream));
}
int nr_impression_metrics(const float* scores, const unsigned char* labels, const long long* seg_offsets, long long n_seg,
                          double* metrics, int* bad_label_flag, void* stream) {
    NR_REQUIRE(scores && labels && seg_offsets && metrics && bad_label_flag && n_seg >= 0,
               "nr_impression_metrics: null operand or n_seg=%lld", n_seg);
    return impression_metrics(scores, labels, seg_offsets, n_seg, metrics, bad_label_flag, as_stream(stream));
}
int nr_impression_ranks(const float* scores, const long long* seg_offsets, long long n_seg, int* ranks, int* bad_score_flag, void* stream) {
    NR_REQUIRE(scores && seg_offsets && ranks && bad_score_flag && n_seg >= 0, "nr_impression_ranks: null operand or n_seg=%lld", n_seg);
    return impression_ranks(scores, seg_offsets, n_seg, ranks, bad_score_flag, as_stream(stream));
}
long long nr_topk_dot_workspace(long long n_users, long long n_news, int D, int k) { return topk_dot_workspace(n_users, n_news, D, k); }
int nr_topk_dot(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D, int k,
                const long long* excl_offsets, const long long* excl_rows, long long* idx, float* score, int* bad_row_flag,
                int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream) {
    NR_REQUIRE(users && news && idx && score && bad_row_flag && bad_score_flag, "nr_topk_dot: null operand");
    return topk_dot(users, n_users, ld_users, news, n_news, ld_news, D, k, excl_offsets, excl_rows, nullptr, 0, nullptr, nullptr,
                    idx, score, bad_row_flag, bad_score_flag, workspace, workspace_bytes, as_stream(stream));
}
int nr_topk_dot_capped(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D,
                       int k, const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category,
                       long long* idx, float* score, int* bad_row_flag, int* bad_score_flag, void* workspace,
                       long long workspace_bytes, void* stream) {
    NR_REQUIRE(users && news && categories && idx && score && bad_row_flag && bad_score_flag, "nr_topk_dot_capped: null operand");
    NR_REQUIRE(max_per_category >= 1, "nr_topk_dot_capped: max_per_category=%d below 1", max_per_category);
    return topk_dot(users, n_users, ld_users, news, n_news, ld_news, D, k, excl_offsets, excl_rows, categories, max_per_category,
                    nullptr, nullptr, idx, score, bad_row_flag, bad_score_flag, workspace, workspace_bytes, as_stream(stream));
}
int nr_topk_dot_ranged(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D,
                       int k, const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category,
                       const long long* row_lo, const long long* row_hi, long long* idx, float* score, int* bad_row_flag,
                       int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream) {
    NR_REQUIRE(users && news && row_lo && row_hi && idx && score && bad_row_flag && bad_score_flag, "nr_topk_dot_ranged: null operand");
    NR_REQUIRE(categories == nullptr || max_per_category >= 1, "nr_topk_dot_ranged: max_per_category=%d below 1", max_per_category);
    return topk_dot(users, n_users, ld_users, news, n_news, ld_news, D, k, excl_offsets, excl_rows, categories, max_per_category,
                    row_lo, row_hi, idx, score, bad_row_flag, bad_score_flag, workspace, workspace_bytes, as_stream(stream));
}
int nr_mmr_rerank(const float* news, long long n_news, int ld_news, int D, const long long* shortlist_idx, const float* shortlist_score,
                  long long n_users, int depth, int k, float lambda, long long* idx, float* score, int* bad_row_flag, void* stream) {
    NR_REQUIRE(news && shortlist_idx && shortlist_score && idx && score && bad_row_flag, "nr_mmr_rerank: null operand");
    return mmr_rerank(news, n_news, ld_news, D, shortlist_idx, shortlist_score, n_users, depth, k, lambda, idx, score, bad_row_flag,
                      as_stream(stream));
}
int nr_list_stats(const float* news, long long n_news, int ld_news, int D, const long long* idx, long long n_rows, int k,
                  const int* categories, const int* ks, int n_ks, double* pair_sum, int* distinct, int* bad_row_flag, void* stream) {
    NR_REQUIRE(news && idx && ks && pair_sum && bad_row_flag, "nr_list_stats: null operand");
    return list_stats(news, n_news, ld_news, D, idx, n_rows, k, categories, ks, n_ks, pair_sum, distinct, bad_row_flag,
                      as_stream(stream));
}
long long nr_pool_ranks_workspace(long long n_rows, long long n_news, int D) { return pool_ranks_workspace(n_rows, n_news, D); }
int nr_pool_ranks(const float* queries, long long n_rows, int ld_queries, const float* news, long long n_news, int ld_news, int D,
                  const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets, const long long* excl_rows,
                  long long* rank, float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
                  long long workspace_bytes, void* stream) {
    NR_REQUIRE(queries && news && tgt_offsets && tgt_rows && rank && score && bad_row_flag && bad_score_flag && target_flag,
               "nr_pool_ranks: null operand");
    return pool_ranks(queries, n_rows, ld_queries, news, n_news, ld_news, D, tgt_offsets, tgt_rows, excl_offsets, excl_rows, nullptr,
                      nullptr, rank, score, bad_row_flag, bad_score_flag, target_flag, workspace, workspace_bytes, as_stream(stream));
}
int nr_pool_ranks_ranged(const float* queries, long long n_rows, int ld_queries, const float* news, long long n_news, int ld_news,
                         int D, const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets,
                         const long long* excl_rows, const long long* row_lo, const long long* row_hi, long long* rank, float* score,
                         int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace, long long workspace_bytes,
                         void* stream) {
    NR_REQUIRE(queries && news && tgt_offsets && tgt_rows && row_lo && row_hi && rank && score && bad_row_flag && bad_score_flag &&
                   target_flag,
               "nr_pool_ranks_ranged: null operand");
    return pool_ranks(queries, n_rows, ld_queries, news, n_news, ld_news, D, tgt_offsets, tgt_rows, excl_offsets, excl_rows, row_lo,
                      row_hi, rank, score, bad_row_flag, bad_score_flag, target_flag, workspace, workspace_bytes, as_stream(stream));
}
long long nr_topk_archive_workspace(long long n_users, int P, long long n_news, int F, int hidden, int k) {
    return topk_archive_workspace(n_users, P, n_news, F, hidden, k);
}
int nr_topk_archive(const float* archive, long long n_users, int P, const float* news, long long n_news, int F, const float* W1,
                    const float* b1, int hidden, const float* w2, const float* b2, int k, const long long* excl_offsets,
                    const long long* excl_rows, const int* categories, int max_per_category, long long* idx, float* score,
                    int* bad_row_flag, int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream) {
    NR_REQUIRE(archive && news && W1 && b1 && w2 && b2 && idx && score && bad_row_flag && bad_score_flag,
               "nr_topk_archive: null operand");
    return topk_archive(archive, n_users, P, news, n_news, F, W1, b1, hidden, w2, b2, k, excl_offsets, excl_rows, categories,
                        max_per_category, nullptr, nullptr, idx, score, bad_row_flag, bad_score_flag, workspace, workspace_bytes,
                        as_stream(stream));
}
int nr_topk_archive_ranged(const float* archive, long long n_users, int P, const float* news, long long n_news, int F,
                           const float* W1, const float* b1, int hidden, const float* w2, const float* b2, int k,
                           const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category,
                           const long long* row_lo, const long long* row_hi, long long* idx, float* score, int* bad_row_flag,
                           int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream) {
    NR_REQUIRE(archive && news && W1 && b1 && w2 && b2 && row_lo && row_hi && idx && score && bad_row_flag && bad_score_flag,
               "nr_topk_archive_ranged: null operand");
    return topk_archive(archive, n_users, P, news, n_news, F, W1, b1, hidden, w2, b2, k, excl_offsets, excl_rows, categories,
                        max_per_category, row_lo, row_hi, idx, score, bad_row_flag, bad_score_flag, workspace, workspace_bytes,
                        as_stream(stream));
}
long long nr_pool_ranks_archive_workspace(long long n_rows, int P, long long n_news, int F, int hidden) {
    return pool_ranks_archive_workspace(n_rows, P, n_news, F, hidden);
}
int nr_pool_ranks_archive(const float* archive, long long n_rows, int P, const float* news, long long n_news, int F, const float* W1,
                          const float* b1, int hidden, const float* w2, const float* b2, const long long* tgt_offsets,
                          const long long* tgt_rows, const long long* excl_offsets, const long long* excl_rows, long long* rank,
                          float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
                          long long workspace_bytes, void* stream) {
    NR_REQUIRE(archive && news && W1 && b1 && w2 && b2 && tgt_offsets && tgt_rows && rank && score && bad_row_flag &&
                   bad_score_flag && target_flag,
               "nr_pool_ranks_archive: null operand");
    return pool_ranks_archive(archive, n_rows, P, news, n_news, F, W1, b1, hidden, w2, b2, tgt_offsets, tgt_rows, excl_offsets,
                              excl_rows, nullptr, nullptr, rank, score, bad_row_flag, bad_score_flag, target_flag, workspace,
                              workspace_bytes, as_stream(stream));
}
int nr_pool_ranks_archive_ranged(const float* archive, long long n_rows, int P, const float* news, long long n_news, int F,
                                 const float* W1, const float* b1, int hidden, const float* w2, const float* b2,
                                 const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets,
                                 const long long* excl_rows, const long long* row_lo, const long long* row_hi, long long* rank,
                                 float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
                                 long long workspace_bytes, void* stream) {
    NR_REQUIRE(archive && news && W1 && b1 && w2 && b2 && tgt_offsets && tgt_rows && row_lo && row_hi && rank && score &&
                   bad_row_flag && bad_score_flag && target_flag,
               "nr_pool_ranks_archive_ranged: null operand");
    return pool_ranks_archive(archive, n_rows, P, news, n_news, F, W1, b1, hidden, w2, b2, tgt_offsets, tgt_rows, excl_offsets,
                              excl_rows, row_lo, row_hi, rank, score, bad_row_flag, bad_score_flag, target_flag, workspace,
                              workspace_bytes, as_stream(stream));
}
long long nr_prediction_line_offsets_workspace(long long n_seg) {
    NR_REQUIRE(n_seg >= 0, "nr_prediction_line_offsets_workspace: n_seg=%lld", n_seg);
    return prediction_scan_bytes(n_seg);
}
int nr_prediction_line_offsets(const long long* impression_ids, const int* ranks, const long long* seg_offsets, long long n_seg,
                               long long* line_offsets, void* workspace, long long workspace_bytes, void* stream) {
    NR_REQUIRE(impression_ids && ranks && seg_offsets && line_offsets && workspace && n_seg >= 0,
               "nr_prediction_line_offsets: null operand or n_seg=%lld", n_seg);
    return prediction_line_offsets(impression_ids, ranks, seg_offsets, n_seg, line_offsets, workspace, workspace_bytes, as_stream(stream));
}
int nr_prediction_text(const long long* impression_ids, const int* ranks, const long long* seg_offsets, long long n_seg,
                       const long long* line_offsets, char* text, void* stream) {
    NR_REQUIRE(impression_ids && ranks && seg_offsets && line_offsets && text && n_seg >= 0,
               "nr_prediction_text: null operand or n_seg=%lld", n_seg);
    return prediction_text(impression_ids, ranks, seg_offsets, n_seg, line_offsets, text, as_stream(stream));
}

int nr_accumulate_ext_grad(float* ext, int rows, int ld, int D, float* dW, float* db, void* stream) {
    NR_REQUIRE(ext && dW && rows >= 0 && D >= 1, "nr_accumulate_ext_grad: null operand");
    return accumulate_ext_grad(ext, rows, ld, D, dW, db, as_stream(stream));
}

// ---- batch feed ------------------------------------------------------------------------------------
int nr_slots_device_readable(const void* const* slots, int n) {
    if (slots == nullptr || n <= 0) return 0;
    return slots_device_readable(slots, n);
}
int nr_pack_slots(const void* const* slots, int n_clicked, int n_candidates, int B, int L, long long* out, void* stream) {
    NR_REQUIRE(slots && out && n_clicked >= 0 && n_candidates >= 0 && B >= 0 && L >= 1, "nr_pack_slots: bad arguments");
    for (int i = 0; i < n_clicked + n_candidates; ++i) NR_REQUIRE(slots[i] != nullptr, "nr_pack_slots: slot %d is null", i);
    prof_context("feed");
    return pack_slots(slots, n_clicked, n_candidates, B, L, out, as_stream(stream));
}
int nr_feed_gather(const nr_feed_field* fields, int n_fields, const int* behaviors, int H, int C, const int* records,
                   const long long* rows, int B, long long* user_out, long long* length_out, long long* clicked_out, void* stream) {
    NR_REQUIRE(n_fields >= 0 && n_fields <= kFeedFields && (fields || n_fields == 0) && H >= 0 && C >= 1 && B >= 0,
               "nr_feed_gather: bad arguments n_fields=%d H=%d C=%d B=%d", n_fields, H, C, B);
    NR_REQUIRE(behaviors && rows && (records || !(user_out || length_out || clicked_out)), "nr_feed_gather: null operand");
    FeedField f[kFeedFields];
    for (int i = 0; i < n_fields; ++i) {
        NR_REQUIRE(fields[i].table && fields[i].out && fields[i].width >= 1, "nr_feed_gather: bad field %d", i);
        f[i] = {.table = fields[i].table, .width = fields[i].width, .out = fields[i].out};
    }
    prof_context("feed");
    return feed_gather(f, n_fields, behaviors, H, C, {.records = records, .user = user_out, .length = length_out, .clicked = clicked_out},
                       rows, B, as_stream(stream));
}
int nr_sample_negatives(const int* cand_rows, const unsigned char* labels, const long long* imp_offsets, long long n_imp,
                        const long long* row_offsets, int K, unsigned long long seed, long long epoch, int* behaviors, int H, void* stream) {
    NR_REQUIRE(cand_rows && labels && imp_offsets && row_offsets && behaviors, "nr_sample_negatives: null operand");
    NR_REQUIRE(K >= 1 && n_imp >= 0 && H >= 0, "nr_sample_negatives: bad arguments K=%d n_imp=%lld H=%d", K, n_imp, H);
    prof_context("feed");
    return sample_negatives(cand_rows, labels, imp_offsets, n_imp, row_offsets, K, seed, epoch, behaviors, H, as_stream(stream));
}

// ---- NRMS encoders ---------------------------------------------------------------------------------
// Q | K | V sections of the projected rows start at columns 0, sec, 2*sec with sec = round_up(d, 8): every section (and so
// every head of every section) has the same 16-byte phase, which the title-level attention kernels rely on.  The packed
// projection operands carry zero rows / columns at the section padding, so the padding columns of Q|K|V are exact zeros.
static int qkv_section(int d) { return (d + 7) & ~7; }
// Every attention kernel of both directions (title-level, head-level, fp32) covers head sizes 2 <= d_k <= 32: a shape outside
// that range is rejected here, before the gather / row conversion and the projection GEMM have written anything.
static int check_mhsa_shape(long long n_seq, int T, int d, int heads, int q, int ldx, int ld3) {
    NR_REQUIRE(n_seq >= 0 && T >= 1 && T <= 64 && d >= 8 && heads >= 1 && d % heads == 0 && q >= 1 && q <= 256,
               "mhsa encoder: bad shape n_seq=%lld T=%d d=%d heads=%d q=%d", n_seq, T, d, heads, q);
    NR_REQUIRE(d / heads >= 2 && d / heads <= 32, "mhsa encoder: head size d_k=%d (d=%d, heads=%d) not in [2, 32]", d / heads, d,
               heads);
    NR_REQUIRE(ldx % 8 == 0 && ldx >= d + 1 && ld3 % 8 == 0 && ld3 >= 3 * qkv_section(d), "mhsa encoder: bad pitches ldx=%d ld3=%d",
               ldx, ld3);
    NR_REQUIRE(n_seq * T < (1ll << 31), "mhsa encoder: too many tokens (%lld)", n_seq * T);
    return 0;
}

// the accurate news variant needs the hi/lo title-level attention kernel and a projection GEMM that can emit the low plane of
// the V section (whole 32-column chunks from column 2*sec: d = 20 and d = 40 have none)
static bool mhsa_accurate_shape(int T, int d, int heads, int ld3, int ldx) {
    if (heads < 1 || d % heads != 0) return false;
    const int sec = qkv_section(d);
    return mhsa_title_fwd_supported(T, d / heads, heads, sec, ld3, ldx) && gemm_store_lo_supported(3 * sec, d, 2 * sec);
}
int nr_mhsa_accurate_supported(int T, int d, int heads) {
    return mhsa_accurate_shape(T, d, heads, (3 * qkv_section(d) + 15) & ~15, (d + 8) & ~7) ? 1 : 0;
}
long long nr_mhsa_encoder_live_bytes(long long n_seq, int T, int d) {
    NR_REQUIRE(n_seq >= 0 && T >= 1 && d >= 1, "nr_mhsa_encoder_live_bytes: n_seq=%lld T=%d d=%d", n_seq, T, d);
    return live_tokens_bytes(n_seq, T, qkv_section(d), (3 * qkv_section(d) + 15) & ~15);
}

// the padding-title buffers of one encoder call, released (stream-ordered) on every way out of it
struct PaddingScope {
    PaddingTitles pt;
    cudaStream_t st;
    ~PaddingScope() { free_padding_titles(pt, st); }
};


// the dense input rows [n_seq][T][d] (+ dense_pos) with the ones column at d, as the hi plane of pitch ld_hi
static Bf16Rows dense_rows(const nr_mhsa_encoder_fwd_args* a, void* hi, int ld_hi) {
    return {.src = a->dense, .n_rows = a->n_seq * a->T, .T = a->T, .D = a->d, .s_seq = a->dense_s_seq, .s_tok = a->dense_s_tok,
            .s_col = a->dense_s_col, .pos = a->dense_pos, .width = a->ldx, .hi = hi, .ld_hi = ld_hi, .ones_col = 1};
}

int nr_mhsa_encoder_fwd(const nr_mhsa_encoder_fwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_mhsa_encoder_fwd: null args");
    NR_PROPAGATE(check_mhsa_shape(a->n_seq, a->T, a->d, a->heads, a->q, a->ldx, a->ld3));
    NR_REQUIRE((a->ids != nullptr) != (a->dense != nullptr), "nr_mhsa_encoder_fwd: exactly one of ids / dense");
    NR_REQUIRE(a->wa_bf16 && a->ba && a->qv && a->C_bf16 && a->w && a->out, "nr_mhsa_encoder_fwd: null operand");
    const bool precise_dense = a->dense != nullptr && a->C_lo_bf16 != nullptr;
    NR_REQUIRE(precise_dense || (a->wqkv_bf16 && a->bqkv && a->X_bf16 && a->QKV_bf16), "nr_mhsa_encoder_fwd: null operand");
    NR_REQUIRE(a->p_drop >= 0.f && a->p_drop < 1.f, "nr_mhsa_encoder_fwd: dropout p=%f", a->p_drop);
    NR_REQUIRE(a->dense_pos == nullptr || a->dense != nullptr, "nr_mhsa_encoder_fwd: dense_pos needs the dense (user-level) variant");
    const int sec = qkv_section(a->d);
    if (a->live != nullptr) {
        NR_REQUIRE(a->ids != nullptr && mhsa_title_fwd_supported(a->T, a->d / a->heads, a->heads, sec, a->ld3, a->ldx) &&
                       (a->V_lo_bf16 == nullptr || mhsa_accurate_shape(a->T, a->d, a->heads, a->ld3, a->ldx)),
                   "nr_mhsa_encoder_fwd: live tokens need the ids variant at the title-level attention kernel's shape");
        NR_REQUIRE(a->live_bytes >= live_tokens_bytes(a->n_seq, a->T, sec, a->ld3), "nr_mhsa_encoder_fwd: live buffer too small (%lld bytes)",
                   a->live_bytes);
    }
    if (a->n_seq == 0) return 0;
    const int M = static_cast<int>(a->n_seq * a->T);
    const cudaStream_t st = as_stream(stream);
    prof_context(a->ids != nullptr ? "news.fwd" : "user.fwd");
    if (a->live != nullptr) {
        // the news encoder over live tokens (LiveTokens, nr_ops.h; about a third of a batch of padded titles and left-padded
        // histories): the gather and the projection write the live tokens' X and Q|K|V rows only, in compact order, and the title
        // attention reads a dead token's Q|K|V from the bias rows.  The context stays in token order.  The backward reuses the
        // compaction, the compact X and the compact Q|K|V.
        NR_REQUIRE(a->table_bf16 && a->bad_id_flag && a->V >= 1 && (a->V_lo_bf16 == nullptr || a->C_lo_bf16 != nullptr),
                   "nr_mhsa_encoder_fwd: table / bad_id_flag missing (or V_lo_bf16 without C_lo_bf16)");
        LiveTokens live;
        NR_PROPAGATE(live_tokens(a->ids, a->n_seq, a->T, a->d, a->table_bf16, a->ldx, a->V, a->bqkv, sec, a->ld3, nullptr, a->ldx, nullptr,
                                 nullptr, a->live, a->live_bytes, &live, st, a->bad_id_flag));
        NR_PROPAGATE(gather_rows(a->ids, M, a->T, a->table_bf16, a->V, a->d, a->ldx, a->X_bf16, a->ldx, 0, DropoutCfg{a->p_drop, a->seed},
                                 a->bad_id_flag, st, &live));
        const bool hilo = a->V_lo_bf16 != nullptr;
        NR_PROPAGATE(gemm_store({.A = a->X_bf16, .M = M, .lda = a->ldx, .W = a->wqkv_bf16, .N = 3 * sec, .ldw = a->ldx, .K = a->d},
                                {.out = a->QKV_bf16, .ld_out = a->ld3, .out_bf16 = 1, .bias = a->bqkv, .lo_out = a->V_lo_bf16,
                                 .ld_lo = hilo ? sec : 0, .lo_col0 = hilo ? 2 * sec : 0, .tile_list = live.tiles}, st));
        {
            ProfScope ps(hilo ? "mhsa_core_fwd_hilo" : "mhsa_core_fwd", static_cast<int>(a->n_seq), a->T, a->d, st);
            NR_PROPAGATE(mhsa_title_fwd(a->QKV_bf16, a->ld3, sec, a->n_seq, a->heads, a->C_bf16, a->ldx, context_dropout(a->p_drop, a->seed),
                                        st, a->V_lo_bf16, hilo ? sec : 0, hilo ? a->C_lo_bf16 : nullptr, nullptr, &live));
        }
        NR_PROPAGATE(gemm_additive_pool(a->C_bf16, M, a->ldx, a->d, a->wa_bf16, a->q, a->ldx, a->ba, a->qv, a->T, a->out, a->d,
                                        a->w, st, hilo ? a->C_lo_bf16 : nullptr));
        return 0;
    }
    if (a->dense != nullptr && a->C_lo_bf16 != nullptr) {
        // precise user encoder (user_encoder.py:15-26 at fp32 accuracy): the input enters as a hi/lo pair against the
        // K-concatenated weights [W | W], Q|K|V stays fp32, the attention runs in fp32, the context leaves as hi/lo planes
        NR_REQUIRE(a->wqkv_kcat_bf16 && a->X_kcat_bf16 && a->QKV_f32 && a->bqkv && a->X_bf16,
                   "nr_mhsa_encoder_fwd: precise dense variant needs wqkv_kcat_bf16 / X_kcat_bf16 / QKV_f32 / bqkv / X_bf16");
        NR_REQUIRE(a->QKV_bf16 == nullptr, "nr_mhsa_encoder_fwd: the precise dense variant writes no bf16 Q|K|V (pass NULL)");
        NR_PROPAGATE(rows_to_bf16(dense_rows(a, a->X_bf16, a->ldx), kRowsToBf16, st));
        // the same rows as [hi | lo] K-concatenated: against [W | W] the GEMM computes (hi + lo) . W^T
        Bf16Rows kcat = dense_rows(a, a->X_kcat_bf16, 2 * a->ldx);
        kcat.lo = static_cast<__nv_bfloat16*>(a->X_kcat_bf16) + a->ldx;
        kcat.ld_lo = 2 * a->ldx;
        NR_PROPAGATE(rows_to_bf16(kcat, kRowsToBf16Hilo, st));
        NR_PROPAGATE(gemm_store({.A = a->X_kcat_bf16, .M = M, .lda = 2 * a->ldx, .W = a->wqkv_kcat_bf16, .N = 3 * sec, .ldw = 2 * a->ldx,
                                 .K = 2 * a->ldx},
                                {.out = a->QKV_f32, .ld_out = 3 * sec, .bias = a->bqkv}, st));
        NR_PROPAGATE(mhsa_f32_fwd(a->QKV_f32, 3 * sec, sec, a->n_seq, a->T, a->heads, a->d / a->heads, a->C_bf16, a->C_lo_bf16, a->ldx, st));
        NR_PROPAGATE(gemm_additive_pool(a->C_bf16, M, a->ldx, a->d, a->wa_bf16, a->q, a->ldx, a->ba, a->qv, a->T, a->out, a->d,
                                        a->w, st, a->C_lo_bf16));
        return 0;
    }
    if (a->ids != nullptr && a->V_lo_bf16 != nullptr) {
        // accurate news encoder on the unfused sequence: V, the attention probabilities and the context travel as hi/lo bf16
        // pairs (the projection GEMM emits the low plane of the V section, the title-level attention kernel splits the
        // probabilities in registers and writes both context planes, the pooled sum reads both)
        NR_REQUIRE(a->C_lo_bf16 != nullptr && a->table_bf16 && a->bad_id_flag && a->V >= 1,
                   "nr_mhsa_encoder_fwd: the accurate variant needs C_lo_bf16 (+ table / bad_id_flag)");
        NR_REQUIRE(mhsa_accurate_shape(a->T, a->d, a->heads, a->ld3, a->ldx),
                   "nr_mhsa_encoder_fwd: the accurate variant needs the title-level attention kernel (T=20, d_k=20, <=15 heads) and a "
                   "chunk-aligned V section (d=%d); see nr_mhsa_accurate_supported", a->d);
        NR_PROPAGATE(gather_rows(a->ids, M, a->T, a->table_bf16, a->V, a->d, a->ldx, a->X_bf16, a->ldx, 0,
                                 DropoutCfg{a->p_drop, a->seed}, a->bad_id_flag, st));
        // padding titles (all ids 0, zero table row 0; ~45 % of a batch of left-padded histories) share one Q|K|V tile: the
        // projection computes only the live 64-row tiles, and the attention reads the shared tile for every padding title
        PaddingScope pad{.st = st};
        NR_PROPAGATE(padding_titles(a->ids, a->n_seq, a->T, a->d, a->table_bf16, a->ldx, a->bqkv, sec, a->ld3, &pad.pt, st));
        NR_PROPAGATE(gemm_store({.A = a->X_bf16, .M = M, .lda = a->ldx, .W = a->wqkv_bf16, .N = 3 * sec, .ldw = a->ldx, .K = a->d},
                                {.out = a->QKV_bf16, .ld_out = a->ld3, .out_bf16 = 1, .bias = a->bqkv, .lo_out = a->V_lo_bf16, .ld_lo = sec,
                                 .lo_col0 = 2 * sec, .tile_list = pad.pt.live}, st));
        {
            ProfScope ps("mhsa_core_fwd_hilo", static_cast<int>(a->n_seq), a->T, a->d, st);
            NR_PROPAGATE(mhsa_title_fwd(a->QKV_bf16, a->ld3, sec, a->n_seq, a->heads, a->C_bf16, a->ldx, context_dropout(a->p_drop, a->seed), st,
                                        a->V_lo_bf16, sec, a->C_lo_bf16, &pad.pt));
        }
        NR_PROPAGATE(gemm_additive_pool(a->C_bf16, M, a->ldx, a->d, a->wa_bf16, a->q, a->ldx, a->ba, a->qv, a->T, a->out, a->d,
                                        a->w, st, a->C_lo_bf16));
        return 0;
    }
    if (a->ids != nullptr) {
        NR_REQUIRE(a->table_bf16 && a->bad_id_flag && a->V >= 1, "nr_mhsa_encoder_fwd: table / bad_id_flag missing");
        NR_PROPAGATE(gather_rows(a->ids, M, a->T, a->table_bf16, a->V, a->d, a->ldx, a->X_bf16, a->ldx, 0,
                                 DropoutCfg{a->p_drop, a->seed}, a->bad_id_flag, st));
    } else {
        NR_PROPAGATE(rows_to_bf16(dense_rows(a, a->X_bf16, a->ldx), kRowsToBf16, st));
    }
    // Q|K|V = X . Wqkv^T + b   (multihead_self.py:53-58)
    NR_PROPAGATE(gemm_store({.A = a->X_bf16, .M = M, .lda = a->ldx, .W = a->wqkv_bf16, .N = 3 * sec, .ldw = a->ldx, .K = a->d},
                            {.out = a->QKV_bf16, .ld_out = a->ld3, .out_bf16 = 1, .bias = a->bqkv}, st));
    // per-head attention (multihead_self.py:15-23), dropout on the context only in the news encoder
    const DropoutCfg cdrop = context_dropout(a->ids != nullptr ? a->p_drop : 0.f, a->seed);
    NR_PROPAGATE(mhsa_core_fwd(a->QKV_bf16, a->ld3, sec, a->n_seq, a->T, a->heads, a->d / a->heads, a->C_bf16, a->ldx, cdrop, st));
    // additive pooling (additive.py:35-53)
    NR_PROPAGATE(gemm_additive_pool(a->C_bf16, M, a->ldx, a->d, a->wa_bf16, a->q, a->ldx, a->ba, a->qv, a->T, a->out, a->d,
                                    a->w, st));
    return 0;
}

// bf16 buffers at the canonical pitches ldq, ldx, ld3, ld3; QKV holds the precise dense forward's recomputed Q|K|V (it keeps
// none) or, in the news variant, the compact copy of X (pitch ldx)
// live: the news variant's LiveTokens buffers (live_tokens_bytes)
struct MhsaBwdWorkspace : WorkspaceLayout {
    float* dscore;
    __nv_bfloat16 *dpre, *dC, *dQKV, *QKV;
    char* live;
    long long live_bytes;
    MhsaBwdWorkspace(void* base, long long n_seq, int T, int d, int q)
        : WorkspaceLayout{static_cast<char*>(base)}, dscore(take<float>(n_seq * T)), dpre(take<__nv_bfloat16>(n_seq * T * round_up(q, 16))),
          dC(take<__nv_bfloat16>(n_seq * T * round_up(d + 1, 8))), dQKV(take<__nv_bfloat16>(n_seq * T * round_up(3 * qkv_section(d), 16))),
          QKV(take<__nv_bfloat16>(n_seq * T * round_up(3 * qkv_section(d), 16))),
          live_bytes(live_tokens_bytes(n_seq, T, qkv_section(d), round_up(3 * qkv_section(d), 16))) {
        live = take<char>(live_bytes);
    }
};
long long nr_mhsa_encoder_bwd_workspace(long long n_seq, int T, int d, int q) { return MhsaBwdWorkspace(nullptr, n_seq, T, d, q).bytes(); }

int nr_mhsa_encoder_bwd(const nr_mhsa_encoder_bwd_args* a, void* stream) {
    NR_REQUIRE(a != nullptr, "nr_mhsa_encoder_bwd: null args");
    NR_PROPAGATE(check_mhsa_shape(a->n_seq, a->T, a->d, a->heads, a->q, a->ldx, a->ld3));
    NR_REQUIRE(a->ldq % 8 == 0 && a->ldq >= a->q, "nr_mhsa_encoder_bwd: ldq=%d", a->ldq);
    NR_REQUIRE(a->ldx == ((a->d + 8) & ~7) && a->ld3 == ((3 * qkv_section(a->d) + 15) & ~15) && a->ldq == ((a->q + 15) & ~15),
               "nr_mhsa_encoder_bwd: pitches must be canonical: ldx=round_up(d+1,8), ld3=round_up(3*round_up(d,8),16), ldq=round_up(q,16)");
    NR_REQUIRE(a->wqkvT_bf16 && a->wa_bf16 && a->waT_bf16 && a->ba && a->qv && a->X_bf16 && a->C_bf16 &&
                   a->w && a->dout && a->dWqkv_ext && a->dWa_ext && a->dqv && a->workspace,
               "nr_mhsa_encoder_bwd: null operand");
    NR_REQUIRE(a->QKV_bf16 != nullptr || (a->wqkv_bf16 != nullptr && a->bqkv != nullptr),
               "nr_mhsa_encoder_bwd: Q|K|V was not saved (precise dense forward): pass wqkv_bf16 / bqkv so that it can be recomputed from X");
    NR_REQUIRE((a->ids != nullptr) ? (a->demb != nullptr) : (a->ddense != nullptr),
               "nr_mhsa_encoder_bwd: missing input-gradient buffer");
    NR_REQUIRE(a->dpos == nullptr || a->ids == nullptr, "nr_mhsa_encoder_bwd: dpos needs the dense (user-level) variant");
    NR_REQUIRE(a->ids == nullptr || a->bqkv != nullptr, "nr_mhsa_encoder_bwd: the news variant needs bqkv (Q|K|V of its padding titles)");
    NR_REQUIRE(a->table_bf16 == nullptr || a->ids != nullptr, "nr_mhsa_encoder_bwd: table_bf16 needs the ids (news) variant");
    const MhsaBwdWorkspace ws(a->workspace, a->n_seq, a->T, a->d, a->q);
    NR_REQUIRE(a->workspace_bytes >= ws.bytes(), "nr_mhsa_encoder_bwd: workspace too small (%lld bytes)", a->workspace_bytes);
    const int sec = qkv_section(a->d);
    const bool title_shape = mhsa_title_bwd_supported(a->T, a->d / a->heads, a->heads, sec, a->ld3, a->ldx, a->ld3);
    if (a->live != nullptr) {
        NR_REQUIRE(a->ids != nullptr && title_shape && a->QKV_bf16 != nullptr,
                   "nr_mhsa_encoder_bwd: live tokens need the ids variant at the title-level attention kernel's shape");
        NR_REQUIRE(a->live_bytes >= live_tokens_bytes(a->n_seq, a->T, sec, a->ld3), "nr_mhsa_encoder_bwd: live buffer too small (%lld bytes)",
                   a->live_bytes);
    }
    if (a->n_seq == 0) return 0;
    const int M = static_cast<int>(a->n_seq * a->T);
    const cudaStream_t st = as_stream(stream);

    prof_context(a->ids != nullptr ? "news.bwd" : "user.bwd");
    const void* QKV = a->QKV_bf16;
    if (QKV == nullptr) {  // the precise dense forward keeps no bf16 Q|K|V: recompute it from the saved rows (multihead_self.py:53-58)
        NR_PROPAGATE(gemm_store({.A = a->X_bf16, .M = M, .lda = a->ldx, .W = a->wqkv_bf16, .N = 3 * sec, .ldw = a->ldx, .K = a->d},
                                {.out = ws.QKV, .ld_out = a->ld3, .out_bf16 = 1, .bias = a->bqkv}, st));
        QKV = ws.QKV;
    }
    // --- additive pooling backward ---
    NR_PROPAGATE(pool_dscore(a->C_bf16, a->ldx, a->d, a->n_seq, a->T, a->w, a->dout, a->d, ws.dscore, st));
    NR_PROPAGATE(gemm_additive_dpre(a->C_bf16, M, a->ldx, a->d, a->wa_bf16, a->q, a->ldx, a->ba, a->qv, ws.dscore, ws.dpre, a->ldq,
                                    a->dqv, st));
    NR_PROPAGATE(gemm_pool_dinput({.A = ws.dpre, .M = M, .lda = a->ldq, .W = a->waT_bf16, .N = a->d, .ldw = a->ldq, .K = a->q},
                                  {.w = a->w, .dout = a->dout, .ldo = a->d, .seg_len = a->T, .dx = ws.dC, .ld_dx = a->ldx,
                                   .drop = context_dropout(a->ids != nullptr ? a->p_drop : 0.f, a->seed)}, st));
    // --- attention backward ---
    // the news variant at the title-level kernel's shape runs the projection backward over live tokens only (id in [1, V), or
    // a nonzero table row 0; about a third of a batch of padded titles and left-padded histories): the attention stores their
    // dQ|dK|dV rows in compact order and sums the dead tokens' rows into the bias column, the dead tokens' only weight-gradient
    // term (their X rows are [0 .. 0, 1]); padding titles read their Q|K|V from the shared bias tile (the accurate forward left
    // their rows unwritten)
    // with the forward's live tokens (a->live) the compaction, the compact X and the compact Q|K|V are the forward's: only the
    // tail rows of the compact dQ|dK|dV need their zeros
    LiveTokens live;
    const bool compact = a->ids != nullptr && title_shape;
    const bool from_fwd = a->live != nullptr;
    if (from_fwd) {
        live = live_tokens_view(a->live, a->n_seq, a->T, sec, a->ld3);
        NR_PROPAGATE(live_zero_tail(live, a->n_seq, a->T, ws.dQKV, a->ld3, st));
    } else if (compact) {
        NR_REQUIRE(a->V >= 1, "nr_mhsa_encoder_bwd: V=%d", a->V);
        NR_PROPAGATE(live_tokens(a->ids, a->n_seq, a->T, a->d, a->table_bf16, a->ldx, a->V, a->bqkv, sec, a->ld3, a->X_bf16, a->ldx, ws.QKV,
                                 ws.dQKV, ws.live, ws.live_bytes, &live, st));
    }
    const TitleBwdLive title_live{.tokens = &live, .dbias = a->dWqkv_ext + a->d, .ld_dbias = a->ldx, .compact_qkv = from_fwd ? 1 : 0};
    NR_PROPAGATE(mhsa_core_bwd(QKV, a->ld3, sec, ws.dC, a->ldx, a->n_seq, a->T, a->heads, a->d / a->heads, ws.dQKV, a->ld3, st,
                               compact ? &title_live : nullptr));
    // --- projection backward: the input first (the embedding gradient is 97 % of a data-parallel step's all-reduce: the
    //     caller's event lets the communication start under the weight-gradient GEMM), then the weights (+bias through the
    //     ones column of X) ---
    if (a->ids != nullptr) {
        NR_REQUIRE(a->V >= 1, "nr_mhsa_encoder_bwd: V=%d", a->V);
        NR_PROPAGATE(gemm_scatter_emb({.A = ws.dQKV, .M = M, .lda = a->ld3, .W = a->wqkvT_bf16, .N = a->d, .ldw = a->ld3, .K = 3 * sec},
                                      {.ids = a->ids, .demb = a->demb, .V = a->V, .drop = {a->p_drop, a->seed}, .drop_ld = a->ldx,
                                       .rows = live.index, .tile_list = live.tiles}, st));
        if (a->emb_grad_ready_event != nullptr) NR_CHECK_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(a->emb_grad_ready_event), st));
    } else {
        NR_PROPAGATE(gemm_store({.A = ws.dQKV, .M = M, .lda = a->ld3, .W = a->wqkvT_bf16, .N = a->d, .ldw = a->ld3, .K = 3 * sec},
                                {.out = a->ddense, .ld_out = a->d}, st));
        // X = dense + pos[t]: the positional gradient is the input gradient summed over the sequences
        if (a->dpos != nullptr) NR_PROPAGATE(sum_over_seq(a->ddense, a->n_seq, static_cast<long long>(a->T) * a->d, a->dpos, st));
    }
    // both weight-gradient GEMMs run AFTER the embedding gradient is complete: together they are the window (~0.4 ms) under which
    // the caller's all-reduce of that gradient hides
    NR_PROPAGATE(gemm_weight_grad(ws.dpre, M, a->q, a->ldq, a->C_bf16, a->d, a->ldx, a->dWa_ext, st));
    // compact: the live tokens' dQ|dK|dV against the compact copy of their X rows (+ bias through its ones column); the
    // forward's X when it ran over live tokens
    NR_PROPAGATE(gemm_weight_grad(ws.dQKV, M, 3 * sec, a->ld3, compact && !from_fwd ? ws.QKV : a->X_bf16, a->d, a->ldx, a->dWqkv_ext, st,
                                  0, live.tiles));
    return 0;
}

}  // extern "C"
