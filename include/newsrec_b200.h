/* newsrec_b200 -- C ABI of the Hopper-native (sm_90a) NRMS / NAML / LSTUR / TANR / Exp1 / Hi-Fi Ark hot path.
 *
 * Drop-in boundary for the reference's Python modules (yusanshi/news-recommendation @ 8323a4f).  The
 * reference has no FFI of its own (pure PyTorch); these are the entry points a maintainer binds with
 * ctypes from src/model/general/**, src/model/<NAME>/{news,user}_encoder.py (see INTEGRATION.md).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; the caller owns every buffer
 *     (PyTorch caching allocator); the library allocates nothing persistent;
 *   - all work is enqueued asynchronously on `stream` (a cudaStream_t passed as void*); no implicit syncs;
 *   - return 0 on success, a positive cudaError_t on a CUDA failure, -1 on an argument/shape violation
 *     (detected before any launch; the Hi-Fi Ark entry points return -2 for a shape outside their stated bounds); nr_last_error() returns the message for the calling thread;
 *   - bf16 operand matrices are row-major with a pitch ("ld", in elements) that is a multiple of 8;
 *     an activation matrix of logical width D carries a constant 1.0 in column D (it turns the next
 *     weight-gradient GEMM's extra column into the bias gradient) and zeros behind it;
 *   - token ids are int64 exactly as the reference's DataLoader produces them; indexing is bit exact;
 *     id 0 is padding_idx: its row is READ like any other (reference behaviour) and its gradient skipped.
 *   - re-entrant; the only global state is a launch counter and the device watchdog record.
 */
#ifndef NEWSREC_B200_H
#define NEWSREC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- library state ------------------------------------------------------------------------------ */
int nr_version(void);                       /* ABI version, currently 1 */
const char* nr_last_error(void);            /* message of the last failing call on this thread */
int nr_device_error(int out4[4]);           /* watchdog record {code, block, thread, aux}; code 0 = none */
long long nr_launch_count(void);            /* kernels this library has launched so far */
int nr_num_sms(void);
/* TRIAGE ONLY (tests): route the GEMMs through a plain SIMT accumulate + the same epilogue functors, to
 * tell a wgmma/TMA pipeline bug from an epilogue bug.  Never enabled by the product path. */
void nr_debug_set_simt_gemm(int on);
/* 1 in a triage build (`make TRIAGE=1`), 0 in the release library, where nr_debug_set_simt_gemm is a no-op, the SIMT
 * kernels are not compiled and no environment switch is consulted on a launch path */
int nr_has_triage_backends(void);
/* Tests (release library too): on != 0 makes nr_gru_fwd run the per-step sequence even where the persistent recurrence applies,
 * on == 0 restores the default.  Until the first call it follows NEWSREC_GRU_STEPWISE (set: per-step), read once. */
void nr_debug_set_gru_stepwise(int on);
/* Tests (release library too): the store GEMM with every option of its epilogue, out[M][N] = act(sum_s A[r + s - tap_origin] .
 * W_s^T + bias) [* (1 - t^2)] [* dropout], fields one for one with the library's internal operands and store configuration.
 * Tap s (taps 1..4) reads weight rows [s * w_tap_rows, + N) against row r + s - tap_origin of A, zero outside [0, M);
 * tap_origin < 0 is taps / 2.  tanh and relu exclude each other; dtanh_src (bf16, pitch dtanh_ld, even; 4-byte aligned) multiplies
 * by 1 - t^2 at the output's own row and column.  The row map sends A row r = s * rm_seg_in + t + rm_in_off to output row
 * s * rm_seg_out + t + rm_out_off when 0 <= t < rm_seg_len (rm_seg_in == 0: identity).  Dropout (p_drop > 0) keys its mask on
 * the output row and column with pitch ld_out.  ones_col >= N (bf16 output, < ld_out): column ones_col = 1 and columns
 * (ones_col, ones_zero_upto) = 0, ones_zero_upto <= ld_out, in mapped rows.  lo_out (bf16 output): columns [lo_col0, N) also
 * leave bf16(y - bf16(y)) at lo_out[row][col - lo_col0], pitch ld_lo.  accumulate (fp32 output): out += result.  out and lo_out
 * must be 16-byte aligned.  Returns -1 before any launch for a configuration the GEMM does not support. */
typedef struct {
    const void* A;
    int M, lda;
    const void* W;
    int N, ldw, K, taps, w_tap_rows, tap_origin;
    void* out;
    int ld_out, out_bf16, relu, tanh;
    const void* dtanh_src;
    int dtanh_ld;
    const float* bias;
    int rm_seg_in, rm_in_off, rm_seg_len, rm_seg_out, rm_out_off;
    float p_drop;
    unsigned long long seed;
    int ones_col, ones_zero_upto;
    void* lo_out;
    int ld_lo, lo_col0, accumulate, rows_per_tile;
} nr_gemm_store_args;
int nr_debug_gemm_store(const nr_gemm_store_args* a, void* stream);
/* TUNING ONLY (tools/kbench.py): dev_buf holds slots x 148 x 16 int64; the k-th gemm_nt planned after this call
 * writes, per CTA, cycle counters into slot k: [0] TMA producer waiting for a free A stage, [1] consumer warpgroups
 * waiting for A data, [4] epilogue body, [5] kernel, [6] tiles.  Null (default) switches the counters off. */
void nr_debug_set_gemm_timing(void* dev_buf, int slots);
/* The live-token compaction of the news encoder's backward (see table_bf16 of nr_mhsa_encoder_bwd_args), on its own: ids
 * [n_seq*T] (T <= 32), the bf16 table (pitch ldx, or NULL) and the gathered rows X [n_seq*T][ldx] in; out the per-title live
 * mask [n_seq] and padding flag [n_seq], the offsets [n_seq+1], the compact -> token index [n_seq*T], the compact tile list
 * [1 + ceil(n_seq*T/64)] (count first), the compact copy of X into Xc [n_seq*T][ldx] and the zero tail rows of Xc and of
 * dqkv_c [n_seq*T][ld3], ld3 = round_up(3*round_up(d, 8), 16).  bqkv [3*round_up(d, 8)]: the padding Q|K|V tile's bias. */
int nr_debug_live_tokens(const long long* ids, long long n_seq, int T, int d, const void* table, int V, const void* X, int ldx,
                         const float* bqkv, unsigned* mask, unsigned char* pad, int* offset, int* index, int* tiles, void* Xc,
                         void* dqkv_c, void* stream);
/* Data parallel: the weight-gradient GEMMs (nr_gemm_tn and the composites' internal calls) leave n SMs free, so that the
 * channel CTAs of a gradient all-reduce running on a side stream have somewhere to run (0 = use every SM, the default). */
void nr_reserve_sms_for_comm(int n);
/* Live per-kernel timing for bench.py: CUDA events on the launching stream around every kernel of this
 * library.  nr_profile_report writes JSON {"<context>/<op>[shape]": [launches, total_ms], ...}, returns its
 * length (or -1 if cap is too small) and clears the records.  Off by default. */
void nr_profile_enable(int on);
void nr_profile_context(const char* ctx);
int nr_profile_report(char* buf, int cap);

/* ---- operand preparation ------------------------------------------------------------------------- */
/* fp32 [R][C] (pitch lds) -> zero padded bf16 [R][ld]; transpose!=0: dst is [C][ld] with dst[c][r]=src[r][c] */
int nr_cast_pad_bf16(const float* src, int R, int C, int lds, void* dst_bf16, int ld, int transpose, void* stream);
/* the same for up to 8 matrices in ONE launch (host arrays of length n; the operands of an encoder are rebuilt together) */
int nr_cast_pad_bf16_many(int n, const float* const* src, const int* R, const int* C, const int* lds, void* const* dst_bf16,
                          const int* ld, const int* transpose, void* stream);
/* fp32 rows [n][D] with element strides -> bf16 [n][ld] + ones column */
int nr_rows_to_bf16(const float* src, long long n, int D, long long s_row, long long s_col, void* dst_bf16, int ld,
                    void* stream);
/* the same rows as a hi/lo bf16 pair in one pass: hi [n][ld] = bf16(x) + ones column at D, lo [n][ld] = bf16(x - hi) with zeros
 * from column D on (input of nr_additive_attention_fwd_hilo) */
int nr_rows_to_bf16_hilo(const float* src, long long n, int D, long long s_row, long long s_col, void* hi_bf16, void* lo_bf16,
                         int ld, void* stream);

/* ---- reference: nn.Embedding lookup (src/model/NRMS/news_encoder.py:38 etc.) --------------------- */
/* X[row(seg,t)] = table[ids[seg*T+t]]; padded!=0 writes the zero-padded CNN layout (T+2 rows per segment).
 * *bad_id_flag (device int) is set to 1 if an id is outside [0,V) (the reference would raise IndexError). */
int nr_gather_rows(const long long* ids, long long n_tok, int T, const void* table_bf16, int V, int D, int ld,
                   void* X_bf16, int padded, float p_drop, unsigned long long seed, int* bad_id_flag, void* stream);

/* ---- reference: nn.Linear / nn.Conv2d(1,F,(3,d)) as a wgmma GEMM with fused bias/ReLU/dropout --- */
/* out[M][N] = act(A . W^T + bias); taps==3: window-3 conv over the padded layout (rows_per_tile = k*(T+2)) */
int nr_linear(const void* A_bf16, int M, int lda, const void* W_bf16, int N, int ldw, int K, int taps, int w_tap_rows,
              int rows_per_tile, const float* bias, int relu, void* out, int ld_out, int out_is_bf16, void* stream);

/* D[Ma][Nb] += A[:, :Ma]^T . B[rows+shift, b_col0:b_col0+Nb]   (weight gradients; fp32 accumulate) */
int nr_gemm_tn(const void* A_bf16, int Kr, int Ma, int lda, const void* B_bf16, int b_rows, int b_cols, int ldb,
               int b_col0, int Nb, int b_row_shift, float* D, int ldd, void* stream);

/* ---- reference: MultiHeadSelfAttention core (src/model/general/attention/multihead_self.py:15-23) -- */
/* Q | K | V sections of a row start at columns 0, sec, 2*sec (sec >= heads*dk; dQ|dK|dV likewise, padding written as zeros).
 * Shape: n_seq >= 0 (0 launches nothing), heads >= 1, 1 <= T <= 64, 2 <= dk <= 32; ld_qkv, ld_dqkv >= 3*sec, ld_ctx >= d+1 (ones
 * column at d, zeros behind it), ld_dctx >= d, every pitch a multiple of 8 (the context dropout mask is the library's hash of
 * row * ld_ctx + col); 0 <= p_drop < 1.  Nothing outside the head columns of qkv and columns [0, d) of dctx reaches a result
 * (NaN there is harmless); dqkv columns [3*sec, ld_dqkv) are not written. */
int nr_mhsa_core_fwd(const void* qkv_bf16, int ld_qkv, int sec, long long n_seq, int T, int heads, int dk, void* ctx_bf16,
                     int ld_ctx, float p_drop, unsigned long long seed, void* stream);
int nr_mhsa_core_bwd(const void* qkv_bf16, int ld_qkv, int sec, const void* dctx_bf16, int ld_dctx, long long n_seq, int T,
                     int heads, int dk, void* dqkv_bf16, int ld_dqkv, void* stream);

/* ---- reference: AdditiveAttention.forward (src/model/general/attention/additive.py:27-53) ----------- */
/* X bf16 [n_seg*seg_len][ldx] (ones column at D) -> out fp32 [n_seg][ldo]; w_out [rows] saved for backward */
int nr_additive_attention_fwd(const void* X_bf16, long long n_seg, int seg_len, int D, int ldx, const void* Wa_bf16,
                              int q, int ldw, const float* ba, const float* qv, float* out, int ldo, float* w_out,
                              void* stream);
/* the same with the input as a hi/lo pair X = X_bf16 + X_lo_bf16 (same pitch; nr_rows_to_bf16_hilo): the scores read the hi
 * plane, the pooled sum both (~16 mantissa bits).  The backward is nr_additive_attention_bwd on the hi plane. */
int nr_additive_attention_fwd_hilo(const void* X_bf16, const void* X_lo_bf16, long long n_seg, int seg_len, int D, int ldx,
                                   const void* Wa_bf16, int q, int ldw, const float* ba, const float* qv, float* out, int ldo,
                                   float* w_out, void* stream);
/* backward.  dX bf16 [rows][ld_dx] (=, columns [D, ld_dx) not written), dWa_ext fp32 [q][ldx] (+=, columns [0, D] only: column D
 * is d(bias)), dqv [q] (+=).  w [rows] is the forward's saved softmax weights, dout fp32 [n_seg][ldo], WaT bf16 [D][ldwT] = Wa^T.
 * Accepted shapes: n_seg >= 0 (0 launches nothing), 1 <= seg_len <= 64 (the forward's limit), 1 <= q <= 256, D >= 4 with
 * D % 4 == 0, and q x D fitting one weight slice of the dPre GEMM (as in the forward); pitches ldx >= D + 1 (the ones column at
 * D, 1.0), ldw >= D, ldwT >= q, ld_dx >= D, each a multiple of 8, and ldo >= D a multiple of 4; bf16 operands, dout and the
 * workspace 16-byte aligned.  Every shape is checked before the first launch: a refused call returns -1 with dX, dWa_ext and
 * dqv untouched.  Nothing outside X's columns [0, D], Wa's columns [0, D), WaT's columns [0, q) and dout's columns [0, D)
 * reaches a result (NaN there is harmless).  dX is the same bits on every run; dWa_ext and dqv are sums of atomic adds.
 * workspace: nr_additive_attention_bwd_workspace(...) bytes: dscore fp32 [rows] at 0, dPre bf16 [rows][round_up(q, 16)] at
 * the next 256-byte boundary. */
long long nr_additive_attention_bwd_workspace(long long n_seg, int seg_len, int q);
int nr_additive_attention_bwd(const void* X_bf16, long long n_seg, int seg_len, int D, int ldx, const void* Wa_bf16,
                              const void* WaT_bf16, int q, int ldw, int ldwT, const float* ba, const float* qv,
                              const float* w, const float* dout, int ldo, void* dX_bf16, int ld_dx, float* dWa_ext,
                              float* dqv, void* workspace, long long workspace_bytes, void* stream);

/* ---- reference: DotProductClickPredictor.forward (src/model/general/click_predictor/dot_product.py) - */
int nr_dot_score_fwd(const float* cand, const float* user, int B, int C, int D, float* logits, void* stream);
int nr_dot_score_bwd(const float* cand, const float* user, const float* dlogits, int B, int C, int D, float* dcand,
                     float* duser, void* stream);

/* ---- reference: src/dataset.py:64-85 + default_collate (the slot-major batch the model receives, src/train.py:183-190) --
   slots[0 .. n_clicked) are the browsed-news tensors, then n_candidates candidate tensors, each int64 [B][L] contiguous and
   readable by the device (device memory or page-locked host memory, nr_slots_device_readable == 1).  One launch writes the
   impression-major block out[(b*n_clicked + h)*L + t], then out[B*n_clicked*L + (b*n_candidates + c)*L + t]. */
int nr_slots_device_readable(const void* const* slots, int n);
int nr_pack_slots(const void* const* slots, int n_clicked, int n_candidates, int B, int L, long long* out, void* stream);

/* ---- device-resident feed (newsrec_b200.feed.DeviceFeed): the parsed news and behaviour tables live on the device and ONE
   launch gathers a batch from them.  Every pointer is device memory.
     behaviors int32 [R][H + C]: the news rows of behaviour row r -- its first H browsed news left-padded with the padding news,
                                 then its C candidates;
     records   int32 [R][2 + C]: user, clicked_news_length (the history length after truncation), the C clicked labels;
     rows      int64 [B]:        the batch's behaviour rows, each in [0, R).
   For each field f, table int32 [n_news][width] (every value of behaviors is a row of it) and out int64 [B*H + B*C][width]:
     out[(b*H + h)*width + t]         = table[behaviors[rows[b]][h]][t]       rows [0, B*H): browsed news, impression-major
     out[(B*H + b*C + c)*width + t]   = table[behaviors[rows[b]][H + c]][t]   then the candidates
   and, each only when not null, user_out[b] = records[rows[b]][0], length_out[b] = records[rows[b]][1] (int64 [B]) and
   clicked_out[c*B + b] = records[rows[b]][2 + c] (int64 [C][B]); records may be null when all three are.  At most 8 fields;
   H >= 0, C >= 1, B >= 0 (0 launches nothing), width >= 1.  Rows are copied with 16-byte stores where width is even and out
   is 16-byte aligned, with 16-byte loads as well where width is a multiple of 4 and table is 16-byte aligned. */
typedef struct {
    const int* table;
    int width;
    long long* out;
} nr_feed_field;
int nr_feed_gather(const nr_feed_field* fields, int n_fields, const int* behaviors, int H, int C, const int* records,
                   const long long* rows, int B, long long* user_out, long long* length_out, long long* clicked_out, void* stream);

/* ---- negative sampling for the device feed (DeviceFeed(..., resample_negatives=True)): ONE launch redraws the candidate
   columns of the behaviour table from MIND's raw impressions, for one (seed, epoch).  Every pointer is device memory.
     cand_rows   int32 [n_cand], labels uint8 [n_cand]: impression i holds candidates [imp_offsets[i], imp_offsets[i+1]); label 1
                 marks a positive, 0 a negative, any other value neither (the reference's endswith('1') / endswith('0'));
     imp_offsets int64 [n_imp + 1];
     row_offsets int64 [n_imp + 1]: impression i owns behaviour rows [row_offsets[i], row_offsets[i+1]), R_i = min(P, floor(N / K))
                 of them for its P positives and N negatives (the reference's balancing count, the same for every draw);
     behaviors   int32 [*][H + 1 + K].
   The draw sorts impression i's negatives by (h_j, j) ascending, j being a negative's ordinal among them (file order) and h_j the
   high 32 bits of
       x = 0;  for v in (seed, epoch, i, j):  x = f((x ^ v) + 0x9E3779B97F4A7C15)          (all uint64, mod 2^64)
       f(z): z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  z ^ (z >> 31)
   (splitmix64's finaliser; epoch as its two's complement).  Owned row p gets behaviors[r][H] = the p-th positive in file order and
   behaviors[r][H + 1 + k] = the negative of sorted place p*K + k, k < K, so no two rows of an impression share a negative.
   Exactly columns H .. H + K of the owned rows are written, and never more than R_i rows of impression i; nothing else (history
   columns, other rows) is touched.  Integer only: the same bits on every run and device.  Any number of candidates per
   impression (fewer than 2^32 negatives); the work is O(N^2 / 32) per lane.  K >= 1, n_imp >= 0 (0 launches nothing), H >= 0. */
int nr_sample_negatives(const int* cand_rows, const unsigned char* labels, const long long* imp_offsets, long long n_imp,
                        const long long* row_offsets, int K, unsigned long long seed, long long epoch, int* behaviors, int H,
                        void* stream);

/* Batched form of the evaluator's scoring loop (src/evaluate.py:245-265 calls get_prediction once per impression and
 * synchronises on .tolist() each time): the news vectors live in ONE device matrix news[n_news][D]; the candidates of
 * impression s are cand[seg_offsets[s] .. seg_offsets[s+1]) (indices into news), user[s] its user vector;
 * scores[i] = news[cand[i]] . user[s].  seg_offsets has n_seg + 1 entries (int64, device), seg_offsets[0] = 0.
 * *bad_id_flag is set if a candidate index is outside [0, n_news). */
int nr_segment_dot(const float* news, long long n_news, int D, const long long* cand, long long n_cand,
                   const long long* seg_offsets, long long n_seg, const float* user, float* scores, int* bad_id_flag,
                   void* stream);

/* The evaluator's metrics (src/evaluate.py:160-168, 267-271: sklearn roc_auc_score + NumPy mrr / nDCG per impression):
 * metrics[s] = {AUC, MRR, nDCG@5, nDCG@10} of impression s, whose candidates are
 * scores[seg_offsets[s] .. seg_offsets[s+1]) with labels (0/1, uint8) at the same positions.  All fp64, [n_seg][4].
 *   place_i = #{j : s_j > s_i} + #{j > i : s_j == s_i}: candidate i's 0-based position in the descending order, ties taken
 *             as the stable reading of argsort(s)[::-1] (among equal scores the later candidate first; -0 == +0);
 *   AUC     = sum_{i pos} (2 #{neg j : s_j < s_i} + #{neg j : s_j == s_i}) / (2 P N)  (Mann-Whitney, counted in integers);
 *   MRR     = sum_{i pos} 1 / (place_i + 1) / P;
 *   nDCG@k  = sum_{i pos, place_i < k} 1 / log2(place_i + 2)  /  sum_{r < min(P, k)} 1 / log2(r + 2).
 * NaN rows: a non-finite score or a label other than 0/1 (all four); P == 0 (all four); N == 0 (AUC only).
 * *bad_label_flag is set if a label is not 0 or 1.  Any segment length works (staged through shared memory in chunks). */
int nr_impression_metrics(const float* scores, const unsigned char* labels, const long long* seg_offsets, long long n_seg,
                          double* metrics, int* bad_label_flag, void* stream);

/* Test-set predictions (the leaderboard's prediction.txt).  Impressions are delimited by seg_offsets as above.
 *   nr_impression_ranks: ranks[i] = place_i + 1 (int32), place_i exactly as nr_impression_metrics defines it, so every
 *     impression's ranks are a permutation of 1..n.  An impression holding a non-finite score sets *bad_score_flag and
 *     gets ranks 0 (its order is undefined).  An impression has fewer than 2^31 candidates.
 *   nr_prediction_line_offsets: line s is "<impression_ids[s]> [r_0,r_1,...,r_{n-1}]\n" in decimal ("<id> []\n" when
 *     empty); writes line_offsets[s] = its first byte (int64, n_seg + 1 entries, line_offsets[n_seg] = the total) with
 *     one length kernel and a CUB exclusive scan in workspace (nr_prediction_line_offsets_workspace(n_seg) bytes, -1 if
 *     the query fails or n_seg >= 2^31 - 1).  impression_ids are int64 and meant to be non-negative (a negative one prints as its unsigned value).
 *   nr_prediction_text: writes the bytes of every line into text[line_offsets[s] .. line_offsets[s + 1]) in one launch.
 * All pointers are device memory.  Null operands or n_seg < 0 return -1 before any launch. */
int nr_impression_ranks(const float* scores, const long long* seg_offsets, long long n_seg, int* ranks, int* bad_score_flag,
                        void* stream);
long long nr_prediction_line_offsets_workspace(long long n_seg);
int nr_prediction_line_offsets(const long long* impression_ids, const int* ranks, const long long* seg_offsets, long long n_seg,
                               long long* line_offsets, void* workspace, long long workspace_bytes, void* stream);
int nr_prediction_text(const long long* impression_ids, const int* ranks, const long long* seg_offsets, long long n_seg,
                       const long long* line_offsets, char* text, void* stream);

/* Recommendation over a whole news pool: the k best news of every user, score[u][n] = users[u] . news[n], without the
 * n_users x n_news score matrix ever reaching memory.  users fp32 [n_users][ld_users], news fp32 [n_news][ld_news] (row
 * pitches in elements, >= D), 1 <= k <= 128, 1 <= D <= 4096, n_users and n_news below 2^31 - 64.  Optional exclusions in CSR
 * form (both null, or both device int64): user u never gets the news rows excl_rows[excl_offsets[u] .. excl_offsets[u + 1])
 * (a set: duplicates and any order are fine; a row outside [0, n_news) sets *bad_row_flag and is otherwise ignored).
 * Outputs idx int64 [n_users][k] and score fp32 [n_users][k], best first: higher score, then lower news row (identical news
 * rows come out in row order); when fewer than k news are eligible the trailing slots hold -1 / -inf.  A non-finite score of
 * any (user, news) pair sets *bad_score_flag (the order is then undefined).  The same inputs give the same bits on every run.
 * Scores: hi/lo bf16 planes of both operands, hi.hi + hi.lo + lo.hi on the tensor cores with fp32 accumulation, within
 *     |score - u.n| <= (2^-15 + 3 round_up(D, 64) 2^-23) sum_i |u_i| |n_i|
 * of the exact dot product of the fp32 inputs.  workspace: nr_topk_dot_workspace(...) bytes (256-byte aligned; -1 for a
 * shape outside the limits above), which depends on the device's SM count.  Every limit is checked before the first launch;
 * n_users == 0 or n_news == 0 launches nothing. */
long long nr_topk_dot_workspace(long long n_users, long long n_news, int D, int k);
int nr_topk_dot(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D, int k,
                const long long* excl_offsets, const long long* excl_rows, long long* idx, float* score, int* bad_row_flag,
                int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream);

/* nr_topk_dot with at most m = max_per_category news of one category per list (diversified recommendation).  categories is
 * device int32 [n_news], one key per news row (any value: 0, negative keys and so on are ordinary keys).  With s(u, n) the bit
 * pattern nr_topk_dot computes for the pair and E_u the pool without u's exclusions: walk E_u in nr_topk_dot's output order
 * (score descending, then lower row) and take a news iff, at that moment, fewer than m taken news share its category and fewer
 * than k news are taken in all.  The output is the taken news in walk order, with nr_topk_dot's shapes and padding: idx int64
 * [n_users][k] and score fp32 [n_users][k], -1 / -inf after the last taken news (a user gets fewer than k news when the caps
 * run out, e.g. with fewer than ceil(k / m) categories).  The result is exact with respect to the kernel's own scores, ties
 * included; excluded news never count against a cap; m >= k gives nr_topk_dot's output bit for bit; the same inputs give the
 * same bits on every run.  The walk is the greedy of a matroid (at most m per category, at most k in all), applied inside the
 * kernel's candidate buffers, so the n_users x n_news score matrix still never reaches memory.  One cap field per call: two
 * simultaneous caps (category and subcategory) are not a matroid and are not supported.  Every limit of nr_topk_dot, a null
 * categories and max_per_category < 1 are refused (-1) before the first launch.  workspace: nr_topk_dot_workspace(...) bytes
 * (the same layout).  Flags as nr_topk_dot. */
int nr_topk_dot_capped(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D,
                       int k, const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category,
                       long long* idx, float* score, int* bad_row_flag, int* bad_score_flag, void* workspace,
                       long long workspace_bytes, void* stream);

/* nr_topk_dot (categories null) or nr_topk_dot_capped (categories non-null, max_per_category >= 1) over a news range per
 * user (recommendation from the news live at each request's time).  row_lo / row_hi are device int64 [n_users], both
 * non-null: news row n is a candidate of user u iff row_lo[u] <= n < row_hi[u].  The outputs equal, bit for bit, those of the
 * unranged call with the rows outside [row_lo[u], row_hi[u]) added to u's exclusions (the same scores, order, caps,
 * padding and determinism).  A range with row_lo[u] < 0, row_hi[u] > n_news or row_lo[u] > row_hi[u] sets *bad_row_flag
 * and gives that user an empty list (-1 / -inf); the other users are unaffected.  A non-finite score of a pair inside its
 * user's range sets *bad_score_flag.  Each block of 64 users streams only the 64-row news tiles its users' ranges touch, so
 * the work follows the ranges' spans: sort users by their ranges to keep a block's ranges close.  Every limit of
 * nr_topk_dot (nr_topk_dot_capped's with categories) and a null row_lo / row_hi are refused (-1) before the first launch.
 * workspace: nr_topk_dot_workspace(...) bytes (the same layout). */
int nr_topk_dot_ranged(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D,
                       int k, const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category,
                       const long long* row_lo, const long long* row_hi, long long* idx, float* score, int* bad_row_flag,
                       int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream);

/* Maximal-marginal-relevance (MMR) re-ranking of nr_topk_dot's shortlists (content-diversified recommendation).  news fp32
 * [n_news][ld_news] (pitch >= D), the pool nr_topk_dot scored; shortlist_idx int64 / shortlist_score fp32 [n_users][depth],
 * nr_topk_dot's output at k = depth.  For user u:
 *   shortlist  C_u = the entries before the first -1 (the live ones, L_u <= depth of them; entries after the first -1 are
 *              ignored), in their order (nr_topk_dot's: score descending, then lower row);
 *   relevance  rel_i = (s_i - s_min) / (s_max - s_min) over C_u, s_i the score bits given; rel_i = 1 for all i when
 *              s_max == s_min.  Dot-product scores have a model-dependent scale, so lambda means the same for every model;
 *   similarity sim(i, j) = the cosine of the fp32 news rows i and j, 0 when either row is all zeros;
 *   greedy     S = {}; for t = 0 .. min(k, L_u) - 1 take the i of C_u \ S that maximises
 *                  obj_i = lambda rel_i - (1 - lambda) max_{j in S} sim(i, j)      (the max over {} is 0),
 *              equal objectives going to the lower shortlist position.
 * Outputs idx int64 [n_users][k] and score fp32 [n_users][k] in pick order; score holds the shortlist's own score bits of
 * the picked rows; the slots after the last pick hold -1 / -inf (nr_topk_dot's shapes and padding).  Exact, bit for bit:
 * lambda = 1 gives nr_topk_dot's k-list (obj is rel exactly, and rel never increases along the shortlist); depth == k gives
 * the shortlist's set, reordered; the same inputs give the same bits on every run.
 * Bounds.  Each block of 64 columns of the live rows is gathered and split into hi/lo bf16 (hi = bf16(x), lo = bf16(x - hi))
 * and the Gram G = hi.lo + lo.hi + hi.hi runs on the tensor cores with fp32 accumulation, so, as for nr_topk_dot's scores,
 *     |G_ij - x_i.x_j| <= eps sum_d |x_id||x_jd| <= eps |x_i||x_j|,    eps = 2^-15 + 3 round_up(D, 64) 2^-23.
 * The norms come from the diagonal (G_ii = |x_i|^2 (1 + t_i), |t_i| <= eps) and sim(i, j) = (G_ji rsqrt(G_jj)) rsqrt(G_ii)
 * in correctly rounded fp32 (0 when G_ii or G_jj is 0), so with c = 2 / (1 - eps), against the exact cosine of the inputs:
 *     e_sim = c eps + 2^-21
 * (the 1 / sqrt((1 + t_i)(1 + t_j)) factor is within eps / (1 - eps) of 1 and the error of G_ij is within eps / (1 - eps) of the
 * cosine's scale after it; four roundings on a value below 1 + c eps add at most 2^-21).  rel and obj are rounded once per
 * operation (no contraction), so against obj evaluated in fp64 on the same score bits, the same fp32 lambda and the exact
 * cosines:
 *     e_obj = (1 - lambda) e_sim + 2^-20,
 * and each pick's fp64 objective is within 2 e_obj of the best remaining one.  The bounds assume finite scores and rows whose
 * squared norms are fp32 normal numbers.  Limits: 1 <= D <= 4096; 1 <= k <= depth <= 128; lambda finite in [0, 1];
 * n_users and n_news in [0, 2^31 - 64).  A live shortlist row outside [0, n_news) sets *bad_row_flag (the user's list is then
 * undefined).  Every limit is refused (-1) before the first launch; n_users == 0 launches nothing.  Runs on the stream given. */
int nr_mmr_rerank(const float* news, long long n_news, int ld_news, int D, const long long* shortlist_idx, const float* shortlist_score,
                  long long n_users, int depth, int k, float lambda, long long* idx, float* score, int* bad_row_flag, void* stream);

/* Statistics of recommendation lists (how similar and how varied each list is).  news fp32 [n_news][ld_news] (pitch >= D);
 * idx int64 [n_rows][k], e.g. nr_topk_dot's, nr_topk_dot_capped's or nr_mmr_rerank's output; categories device int32
 * [n_news] (any values) or null; ks a HOST array of n_ks cut-offs, strictly ascending, each in [1, k], n_ks <= 8.  For row r
 * the live entries are those before the first -1 (entries after it are ignored), L_r of them; for cut-off K, K' = min(K, L_r):
 *   pair_sum[r][c] = sum_{j < K'} ( sum_{i < j} sim(i, j) )     (fp64 [n_rows][n_ks]; each inner sum in fp64 with i
 *                    ascending, the outer sum in fp64 with j ascending; 0 when K' < 2)
 *   distinct[r][c] = the number of distinct categories values among the first K' entries   (int32 [n_rows][n_ks], exact)
 * with K = ks[c].  sim is nr_mmr_rerank's cosine, computed the same way by the same device routines: the rows gathered into
 * hi/lo bf16 planes 64 columns at a time, G = hi.lo + lo.hi + hi.hi on the tensor cores with fp32 accumulation,
 * sim(i, j) = (G_ji rsqrt(G_jj)) rsqrt(G_ii) in correctly rounded fp32, 0 when either row is all zeros.  So each pair is
 * within nr_mmr_rerank's
 *     e_sim = c eps + 2^-21,    c = 2 / (1 - eps),    eps = 2^-15 + 3 round_up(D, 64) 2^-23
 * of the exact cosine of the fp32 rows (rows whose squared norms are fp32 normal numbers), and with P = K'(K' - 1) / 2 pairs,
 *     |pair_sum - sum of the exact cosines| <= P e_sim + P^2 2^-52     (the second term: the fp64 additions),
 * so the mean over the pairs is within e_sim + P 2^-52 of the exact mean.  distinct is null iff categories is null.
 * Limits: 1 <= D <= 4096; 1 <= k <= 128; ks as above; n_rows and n_news in [0, 2^31 - 64).  A live entry outside
 * [0, n_news) sets *bad_row_flag (that row's outputs are then undefined).  Every limit is refused (-1) before the first
 * launch; n_rows == 0 launches nothing.  The same inputs give the same bits on every run.  One block per row. */
int nr_list_stats(const float* news, long long n_news, int ld_news, int D, const long long* idx, long long n_rows, int k,
                  const int* categories, const int* ks, int n_ks, double* pair_sum, int* distinct, int* bad_row_flag, void* stream);

/* Ranks over a whole news pool under nr_topk_dot's scores.  Query row q (queries fp32 [n_rows][ld_queries]) has the target
 * set T_q = tgt_rows[tgt_offsets[q] .. tgt_offsets[q + 1]) and the exclusion set X_q (excl_offsets / excl_rows as in
 * nr_topk_dot: both null, or both device int64; a set, any length, order or duplicates).  For every target t of q:
 *     rank(q, t) = |{ n in [0, n_news) \ X_q \ T_q : s(q, n) > s(q, t)  or  (s(q, n) == s(q, t) and n < t) }|
 * where s is bit for bit the score nr_topk_dot computes for the pair (the same planes and tile code): rank(q, t) is t's 0-based
 * position in the order nr_topk_dot returns over the pool without X_q and T_q.  A target is ranked even when it is also in X_q.
 * rank int64 and score fp32 (s(q, t)) are written in target order, [tgt_offsets[0] .. tgt_offsets[n_rows]).  The same inputs
 * give the same bits on every run.  Limits: 1 <= D <= 4096, 0 <= n_rows and 1 <= n_news, both below 2^31 - 64, pitches >= D;
 * at most 32 targets per row: a row with more sets *target_flag and gets rank -1 (score NaN).  A target or exclusion outside
 * [0, n_news) sets *bad_row_flag (such a target's row gets rank -1); a non-finite score of a row with targets sets
 * *bad_score_flag (its ranks are then undefined).  With |s(q, n) - S(n)| <= e(n) (the bound of nr_topk_dot,
 * e(n) = (2^-15 + 3 round_up(D, 64) 2^-23) sum_i |q_i| |n_i|, S(n) the exact dot product of the fp32 inputs):
 *     |{n eligible : S(n) - S(t) > e(n) + e(t)}|  <=  rank(q, t)  <=  |{n eligible : S(n) - S(t) >= -(e(n) + e(t))}|
 * workspace: nr_pool_ranks_workspace(...) bytes (256-byte aligned; -1 for a shape outside the limits), which depends on the
 * device's SM count.  Every limit is checked before the first launch; n_rows == 0 launches nothing. */
long long nr_pool_ranks_workspace(long long n_rows, long long n_news, int D);
int nr_pool_ranks(const float* queries, long long n_rows, int ld_queries, const float* news, long long n_news, int ld_news, int D,
                  const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets, const long long* excl_rows,
                  long long* rank, float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
                  long long workspace_bytes, void* stream);

/* nr_pool_ranks over a news range per query row: row_lo / row_hi device int64 [n_rows], both non-null, and row q counts only
 * news rows n with row_lo[q] <= n < row_hi[q].  rank and score equal, bit for bit, those of nr_pool_ranks with the rows
 * outside [row_lo[q], row_hi[q]) added to X_q.  A target outside its row's range is still ranked, against the row's eligible
 * news (as a target in X_q is).  A range with row_lo[q] < 0, row_hi[q] > n_news or row_lo[q] > row_hi[q] sets
 * *bad_row_flag and gives that row's targets rank -1 (score NaN); the other rows are unaffected.  Only the news tiles that
 * hold a block's targets and that its rows' ranges touch are streamed.  Limits and workspace as nr_pool_ranks'; a null
 * row_lo / row_hi is refused (-1) before the first launch. */
int nr_pool_ranks_ranged(const float* queries, long long n_rows, int ld_queries, const float* news, long long n_news, int ld_news,
                         int D, const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets,
                         const long long* excl_rows, const long long* row_lo, const long long* row_hi, long long* rank, float* score,
                         int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace, long long workspace_bytes,
                         void* stream);

/* Recommendation over a whole news pool under the archive DNN click score of Hi-Fi Ark and DKN (the scorer of
 * nr_archive_score_fwd).  archive fp32 [n_users][P][F] contiguous (DKN: P = 1, the user vector), news fp32 [n_news][F]
 * contiguous, W1 fp32 [hidden][2F] over [c; u], b1 [hidden], w2 [hidden], b2 [1], all device.  For user u and news c:
 *     w = softmax_p(A_u[p] . c)   (P = 1: w = 1 exactly),   score = b2 + sum_j w2_j relu(X_j + sum_p w_p Y_pj)
 *     X = W1[:, :F] c + b1,   Y_p = W1[:, F:] A_u[p]
 * Exclusions, categories (nullable) / max_per_category (>= 1 with categories), outputs, padding, ordering, flags and
 * determinism are nr_topk_dot's (nr_topk_dot_capped's with categories), with these scores in place of the dot products.
 * One routine computes every pair's score in a fixed operation order, so a pair's score is the same bits in nr_topk_archive
 * and nr_pool_ranks_archive and does not depend on k, the cap, the split count or where the user sits in the call.
 * Computation: X and Y in fp32 on the CUDA cores (sequential fma over f, then + b1); the P logits on the tensor cores from
 * hi/lo bf16 planes, as nr_topk_dot's scores; m = max_p l_p, e_p = __expf(l_p - m), z = sum_p e_p (in p order),
 * w_p = e_p rcp(z); pre_j = fma over p of w_p Y_pj onto X_j; out = fma over j of w2_j relu(pre_j) onto b2.
 * Bound.  With L_p, W_p, X_j, Y_pj, pre_j the exact values from the fp32 inputs, u = 2^-24, g(n) = n u / (1 - n u):
 *   logits   |l_p - L_p| <= d_p = (2^-15 + 3 round_up(F, 64) 2^-23) sum_f |A_pf| |c_f|         (nr_topk_dot, per head)
 *   softmax  sum_p |w_p - W_p| <= e_w = (1 + 2^-10) (2 max_p d_p + 2 sum_p W_p (2 + 2 |L_p - L_max| + 4 max_p d_p) 2^-23
 *                                                    + g(P + 2))
 *            (a logit shift moves the softmax by at most 2 max_p d_p in l1; __expf(x) is within 2 + 1.173 |x| ulp of e^x and
 *            the subtraction adds |x| u; each relative error enters w_p and z; the sum, the reciprocal and the product add
 *            g(P + 2); the factor covers the second-order terms)
 *   X, Y     |dX_j| <= g(F + 1) (sum_f |W1_jf| |c_f| + |b1_j|),   |dY_pj| <= g(F) sum_f |W1_j,F+f| |A_pf|
 *   mix      |pre_j - PRE_j| <= E_j = |dX_j| + sum_p W_p |dY_pj| + e_w max_p (|Y_pj| + |dY_pj|)
 *                                   + g(P) (|X_j| + |dX_j| + sum_p (W_p + e_w)(|Y_pj| + |dY_pj|))
 *   output   e = sum_j |w2_j| E_j + g(hidden) (|b2| + sum_j |w2_j| (|PRE_j| + E_j))      (relu is 1-Lipschitz)
 * so |score - SCORE| <= e per pair, SCORE the exact score of the fp32 inputs (finite inputs; normal-range exponentials).
 * The rank band of nr_pool_ranks carries over with this e(n).  Limits: 1 <= k <= 128, 1 <= P <= 32, 1 <= hidden <= 32,
 * 1 <= F <= 4096, n_users P and n_news below 2^31 - 64.  Every limit is refused (-1) before the first launch; n_users == 0
 * or n_news == 0 launches nothing.  workspace: nr_topk_archive_workspace(...) bytes (256-byte aligned; -1 outside the
 * limits), which depends on the device's SM count. */
long long nr_topk_archive_workspace(long long n_users, int P, long long n_news, int F, int hidden, int k);
int nr_topk_archive(const float* archive, long long n_users, int P, const float* news, long long n_news, int F, const float* W1,
                    const float* b1, int hidden, const float* w2, const float* b2, int k, const long long* excl_offsets,
                    const long long* excl_rows, const int* categories, int max_per_category, long long* idx, float* score,
                    int* bad_row_flag, int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream);

/* nr_topk_archive over a news range per user: row_lo / row_hi, the contract (the unranged outputs with the complement of
 * each range added to the exclusions, bit for bit), bad ranges and flags as nr_topk_dot_ranged's.  Limits and workspace as
 * nr_topk_archive's; a null row_lo / row_hi is refused (-1) before the first launch. */
int nr_topk_archive_ranged(const float* archive, long long n_users, int P, const float* news, long long n_news, int F,
                           const float* W1, const float* b1, int hidden, const float* w2, const float* b2, int k,
                           const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category,
                           const long long* row_lo, const long long* row_hi, long long* idx, float* score, int* bad_row_flag,
                           int* bad_score_flag, void* workspace, long long workspace_bytes, void* stream);

/* nr_pool_ranks under nr_topk_archive's scores (the same bits per pair): targets, exclusions, 32-target rows, flags and the
 * rank definition are nr_pool_ranks'; archive [n_rows][P][F] as nr_topk_archive's, one archive per query row.  The band
 * holds with nr_topk_archive's e(n).  Limits as nr_topk_archive's without k, with 1 <= n_news.  workspace:
 * nr_pool_ranks_archive_workspace(...) bytes (256-byte aligned; -1 outside the limits). */
long long nr_pool_ranks_archive_workspace(long long n_rows, int P, long long n_news, int F, int hidden);
int nr_pool_ranks_archive(const float* archive, long long n_rows, int P, const float* news, long long n_news, int F, const float* W1,
                          const float* b1, int hidden, const float* w2, const float* b2, const long long* tgt_offsets,
                          const long long* tgt_rows, const long long* excl_offsets, const long long* excl_rows, long long* rank,
                          float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
                          long long workspace_bytes, void* stream);

/* nr_pool_ranks_archive over a news range per query row: row_lo / row_hi, the contract, targets outside the range and bad
 * ranges as nr_pool_ranks_ranged's.  Limits and workspace as nr_pool_ranks_archive's; a null row_lo / row_hi is refused
 * (-1) before the first launch. */
int nr_pool_ranks_archive_ranged(const float* archive, long long n_rows, int P, const float* news, long long n_news, int F,
                                 const float* W1, const float* b1, int hidden, const float* w2, const float* b2,
                                 const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets,
                                 const long long* excl_rows, const long long* row_lo, const long long* row_hi, long long* rank,
                                 float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
                                 long long workspace_bytes, void* stream);

/* Host-side glue of the weight-gradient GEMMs (nr_gemm_tn with the ones column): ext is [rows][ld] fp32 whose columns
 * [0,D) hold dW and column D holds db.  Adds them into the parameters' own gradient storage (dW [rows][D] contiguous,
 * db [rows] or null) and CLEARS ext, so the caller can keep it as a persistent accumulator across steps. */
int nr_accumulate_ext_grad(float* ext, int rows, int ld, int D, float* dW, float* db, void* stream);

/* ---- reference: NRMS NewsEncoder.forward / UserEncoder.forward -------------------------------------
 *   news  (src/model/NRMS/news_encoder.py:27-48): embedding -> dropout -> MHSA -> dropout -> additive pool
 *   user  (src/model/NRMS/user_encoder.py:15-26): MHSA -> additive pool over dense fp32 news vectors     */
typedef struct {
    long long n_seq;          /* titles (news) or users                                             */
    int T;                    /* tokens per title / history length                                  */
    int d;                    /* model width (word_embedding_dim)                                   */
    int heads;                /* num_attention_heads, d % heads == 0, head size 2 <= d/heads <= 32 (else -1 before any launch) */
    int q;                    /* query_vector_dim                                                   */
    int ldx;                  /* pitch of X / C / weight operands: multiple of 8, >= d+1            */
    int ld3;                  /* pitch of Q|K|V rows: round_up(3*sec, 16), sec = round_up(d, 8): sections at columns 0, sec, 2*sec;
                                 packed weights / biases carry zero rows at the section padding */
    /* input: ids+table (news encoder) or dense (user encoder) */
    const long long* ids;     /* [n_seq*T] or NULL                                                  */
    const void* table_bf16;   /* [V][ldx]                                                           */
    int V;
    const float* dense;       /* fp32 [n_seq][T][d] with element strides below, or NULL             */
    long long dense_s_seq, dense_s_tok, dense_s_col;
    /* parameters as prepared operands */
    const void* wqkv_bf16;    /* [3*sec][ldx]  rows = W_Q | 0 | W_K | 0 | W_V | 0 (zero rows at the section padding) */
    const float* bqkv;        /* [3*sec]       b_Q | 0 | b_K | 0 | b_V | 0                                         */
    const void* wa_bf16;      /* [q][ldx]                                                           */
    const float* ba;          /* [q]                                                                */
    const float* qv;          /* [q]                                                                */
    float p_drop;             /* dropout_probability when training, else 0                          */
    unsigned long long seed;
    /* outputs; X/QKV/C/w are what backward needs (the caller keeps them alive) */
    void* X_bf16;             /* [n_seq*T][ldx]                                                     */
    void* QKV_bf16;           /* [n_seq*T][ld3]; the accurate news variant leaves the rows of 64-row tiles that hold only
                                 padding titles (all ids 0, zero table row 0) unwritten, and V_lo_bf16 likewise            */
    void* C_bf16;             /* [n_seq*T][ldx]                                                     */
    float* w;                 /* [n_seq*T] additive-attention weights                               */
    float* out;               /* [n_seq][d] fp32                                                    */
    int* bad_id_flag;         /* device int, set if an id is out of range                           */
    /* low plane of the context (precise variants below): the pooled sum uses C_bf16 + C_lo_bf16 */
    void* C_lo_bf16;             /* [n_seq*T][ldx]                                                      */
    /* precise DENSE variant (user encoder of the precise mode; selected by dense != NULL and C_lo_bf16 != NULL): the fp32
     * input enters the projection as a hi/lo bf16 pair against K-concatenated weights, Q|K|V stays fp32, the attention runs
     * in fp32 on the CUDA cores, the context leaves as hi (C_bf16) + lo (C_lo_bf16) planes.  QKV_bf16 must be NULL. */
    const void* wqkv_kcat_bf16;  /* [3*sec][2*ldx]: rows as wqkv_bf16; columns [0,d) = W, [ldx, ldx+d) = W again, zeros elsewhere */
    void* X_kcat_bf16;           /* [n_seq*T][2*ldx] workspace: hi | lo operand rows                                   */
    float* QKV_f32;              /* [n_seq*T][3*sec] workspace                                                           */
    /* accurate NEWS variant on the unfused kernels (selected by ids != NULL and V_lo_bf16 != NULL; needs C_lo_bf16 and
     * nr_mhsa_accurate_supported): V, the attention probabilities and the context are hi/lo bf16 pairs; X_bf16 and QKV_bf16
     * (the hi planes) are written as usual and saved for the backward. */
    void* V_lo_bf16;             /* [n_seq*T][sec] low plane of the V section                                            */
    /* dense variants only (NULL otherwise): fp32 [T][d] contiguous positional addend; the rows entering the projection are
     * X = dense + dense_pos[t], summed in fp32 before any rounding (Exp1's user encoder) */
    const float* dense_pos;
    /* ids variant at the title-level attention kernel's shape (T = 20, d_k = 20, <= 15 heads), either precision: NULL, or a
     * buffer of nr_mhsa_encoder_live_bytes(n_seq, T, d) bytes (16-byte aligned) that selects the forward over live tokens
     * (id in [1, V), or every token when row 0 of the table is nonzero).  X_bf16, QKV_bf16 and V_lo_bf16 then hold the live
     * tokens' rows only, in ascending token order, followed by zero X rows up to the next multiple of 64 (below n_seq*T);
     * C_bf16 / C_lo_bf16, w and out are as without it.  The buffer, X_bf16 and QKV_bf16 go to the backward together
     * (nr_mhsa_encoder_bwd_args.live).  Anywhere else a non-NULL live is refused (-1) before any launch. */
    void* live;
    long long live_bytes;
} nr_mhsa_encoder_fwd_args;
int nr_mhsa_accurate_supported(int T, int d, int heads); /* 1: the accurate news variant exists for this shape */
long long nr_mhsa_encoder_live_bytes(long long n_seq, int T, int d); /* bytes of the live-token buffer of the two calls */
int nr_mhsa_encoder_fwd(const nr_mhsa_encoder_fwd_args* a, void* stream);

typedef struct {
    long long n_seq;
    int T, d, heads, q, ldx, ld3, ldq;   /* ldq: pitch of dPre / WaT = round_up(q, 16)                   */
    const long long* ids;                /* NULL for the dense (user) variant                            */
    int V;
    const void* wqkvT_bf16;              /* [d][ld3]  = (W_Q|0|W_K|0|W_V|0)^T                               */
    const void* wa_bf16;                 /* [q][ldx]                                                     */
    const void* waT_bf16;                /* [d][ldq]                                                     */
    const float* ba;
    const float* qv;
    float p_drop;
    unsigned long long seed;
    const void* X_bf16;
    const void* QKV_bf16;
    const void* C_bf16;
    const float* w;
    const float* dout;                   /* [n_seq][d] fp32                                              */
    /* gradients */
    float* dWqkv_ext;                    /* [3*sec][ldx] (+=)  sectioned rows as wqkv_bf16, column d = d(bias); the padding
                                            rows receive exact zeros                                      */
    float* dWa_ext;                      /* [q][ldx]  (+=)  column d = d(bias)                           */
    float* dqv;                          /* [q] (+=)                                                     */
    float* demb;                         /* [V][d] (+=) embedding gradient (ids variant)                 */
    float* ddense;                       /* [n_seq*T][d] (=) input gradient (dense variant)              */
    void* workspace;
    long long workspace_bytes;
    /* QKV_bf16 == NULL (the precise dense forward keeps no bf16 Q|K|V): recomputed here from X_bf16 with these operands */
    const void* wqkv_bf16;               /* [3*sec][ldx] (sectioned, as in the forward arguments)        */
    const float* bqkv;                   /* [3*sec]; also required by the ids variant: the Q|K|V of its padding titles */
    /* optional cudaEvent_t recorded on `stream` as soon as demb is complete (before the weight-gradient GEMM): a data-
     * parallel caller starts the embedding-gradient all-reduce on a side stream that waits for it */
    void* emb_grad_ready_event;
    /* dense variant only (NULL otherwise): fp32 [T][d] (+=) gradient of dense_pos = sum over the sequences of ddense, in a fixed
     * order (bit-identical across runs) */
    float* dpos;
    /* ids variant: the bf16 table of the forward (pitch ldx).  The projection backward runs over the live tokens only -- id in
     * [1, V), or every token when row 0 of the table is nonzero -- and, like the accurate forward, takes a title without one
     * for padding.  NULL: the same verdict from the gathered rows X instead (a token is live when its id is in [1, V) or its
     * row of X is nonzero below column d), which costs a read of the dead tokens' rows.  NULL for the dense variant. */
    const void* table_bf16;
    /* the forward's live-token buffer (nr_mhsa_encoder_fwd_args.live), or NULL: X_bf16 / QKV_bf16 are the forward's compact
     * rows, and the backward reuses its compaction instead of classifying the tokens again */
    void* live;
    long long live_bytes;
} nr_mhsa_encoder_bwd_args;
long long nr_mhsa_encoder_bwd_workspace(long long n_seq, int T, int d, int q);
int nr_mhsa_encoder_bwd(const nr_mhsa_encoder_bwd_args* a, void* stream);

/* ---- reference: title / abstract CNN encoder ------------------------------------------------------------
 *   NAML  TextEncoder      src/model/NAML/news_encoder.py:21-37
 *   LSTUR title branch     src/model/LSTUR/news_encoder.py:56-72
 *   TANR  NewsEncoder      src/model/TANR/news_encoder.py:40-52
 * embedding -> dropout -> Conv2d(1, F, (w, d), padding ((w-1)/2, 0)) -> ReLU -> dropout -> additive pooling, window w = 1 .. 4.
 * With p = (w-1)/2 a segment has L = T + 2p - w + 1 output positions (T at odd w, T-1 at even w).  The conv is w row-shifted
 * wgmma GEMM taps over a zero-padded layout (T+2 rows per segment, token t at row t+1), output j reading rows j+1-p+s, s < w.
 * Shapes: 1 <= T <= 64 (the pooling tile holds whole segments), T >= w - 2p (T >= 2 at an even window), d and F multiples of
 * 4, d, F >= 8, 1 <= q <= 256; both entry points reject any other shape or window with -1 before the first launch. */
typedef struct {
    long long n_seq;
    int T, d, F, q, ldx, ldf;       /* ldx = round_up(d+1, 8), ldf = round_up(F+1, 8)                       */
    const long long* ids;           /* [n_seq*T]                                                          */
    const void* table_bf16;         /* [V][ldx]                                                           */
    int V;
    const void* wconv_bf16;         /* [w*F][ldx]; rows s*F..(s+1)*F hold tap s = weight[:, 0, s, :]        */
    const float* bconv;             /* [F]                                                                */
    const void* wa_bf16;            /* [q][ldf]                                                           */
    const float* ba;
    const float* qv;
    float p_drop;
    unsigned long long seed;
    void* Xp_bf16;                  /* [n_seq*(T+2)][ldx]  gathered rows, zero-padded layout (saved)        */
    void* Y_bf16;                   /* [n_seq*L][ldf]      relu(conv) rows (saved)                          */
    float* w;                       /* [n_seq*L]                                                          */
    float* out;                     /* [n_seq][F]                                                         */
    int* bad_id_flag;
    void* Y_lo_bf16;          /* optional [n_seq*L][ldf]: low plane of the conv output (accurate mode: the pooled sum reads Y + Y_lo) */
    int window;                     /* conv window w, 1 .. 4; 0 means 3 (the reference default)            */
} nr_cnn_encoder_fwd_args;
int nr_cnn_encoder_fwd(const nr_cnn_encoder_fwd_args* a, void* stream);

typedef struct {
    long long n_seq;
    int T, d, F, q, ldx, ldf, ldq;
    const long long* ids;
    int V;
    const void* wconvT_bf16;        /* [w*d][ldf]; rows s*d..(s+1)*d hold (weight[:, 0, w-1-s, :])^T        */
    const void* wa_bf16;            /* [q][ldf]                                                           */
    const void* waT_bf16;           /* [F][ldq]                                                           */
    const float* ba;
    const float* qv;
    float p_drop;
    unsigned long long seed;
    const void* Xp_bf16;
    const void* Y_bf16;
    const float* w;
    const float* dout;              /* [n_seq][F]                                                         */
    float* dWconv_ext;              /* [w][F][ldx] (+=); column d of tap p = (w-1)/2 is d(bias)             */
    float* dWa_ext;                 /* [q][ldf] (+=); column F is d(bias)                                   */
    float* dqv;                     /* [q] (+=)                                                           */
    float* demb;                    /* [V][d] (+=)                                                        */
    void* workspace;
    long long workspace_bytes;
    int window;                     /* as in the forward: 1 .. 4, 0 means 3                               */
} nr_cnn_encoder_bwd_args;
long long nr_cnn_encoder_bwd_workspace(long long n_seq, int T, int F, int q);
int nr_cnn_encoder_bwd(const nr_cnn_encoder_bwd_args* a, void* stream);

/* ---- reference: DKN's knowledge-aware CNN (src/model/DKN/KCNN.py), without context embeddings --------------
 * word embedding | tanh(entity embedding . M + b) stacked as two channels -> Conv2d(2, F, (x, d)) for every window x, no
 * padding (T + 1 - x positions) -> ReLU -> ONE additive attention shared by the windows -> the windows' outputs side by side.
 * Layouts (bf16 rows, 16-byte sections):
 *   X2   [n_seq*T][ldx]   ldx = 2 sec, sec = round_up(d+1, 8): [word (d) | 1 | 0..] [tanh entity (d) | 1 | 0..] (saved)
 *   E    [n_seq*T][lde]   lde = round_up(de+1, 8): gathered entity rows (saved)
 *   Y    window w's relu(conv) rows [n_seq*(T+1-x_w)][ldf], ldf = round_up(F+1, 8), the windows back to back (saved); w likewise
 *   out  [n_seq][ldo] fp32, ldo = n_win * Fs, Fs = round_up(F, 4): window w in columns [w Fs, w Fs + F), the rest 0 (=)
 * Each conv is one wgmma GEMM of x_w row-shifted taps over the compact rows of X2.  The backward puts dY of every window into
 * one [n_seq*T][n_win*ldf] block and runs the transposed conv of all windows as max(x) taps, split into the word half (scattered
 * into dword) and the entity half (times 1 - t^2 -> dZ, then dM and dentity).  Row 0 of both tables is read as stored and gets
 * no gradient (padding_idx).  dout's padding columns must be 0.
 * Shapes: 1 <= n_win <= 4, 1 <= x_w <= 4, max(x) <= T <= 64, d and de multiples of 4 (>= 8), F even (>= 8), 1 <= q <= 256; both
 * entry points reject any other shape with -1 before the first launch. */
typedef struct {
    long long n_seq;
    int T, d, de, F, q, n_win;
    int win[4];
    int ldx, lde, ldf, ldo;
    const long long* word_ids;      /* [n_seq*T]                                                          */
    const long long* entity_ids;    /* [n_seq*T]                                                          */
    const void* word_table_bf16;    /* [V][sec]                                                           */
    int V;
    const void* entity_table_bf16;  /* [Ve][lde]                                                          */
    int Ve;
    const void* mT_bf16;            /* [d][lde]  transform_matrix^T                                       */
    const float* mb;                /* [d]       transform_bias                                           */
    const void* wconv_bf16;         /* [sum x_w * F][ldx]; window w, tap s at rows (x_0 + .. + x_(w-1) + s) F, in X2's columns */
    const float* bconv;             /* [n_win * F]                                                        */
    const void* wa_bf16;            /* [q][ldf]                                                           */
    const float* ba;
    const float* qv;
    void* X2_bf16;
    void* E_bf16;
    void* Y_bf16;
    float* w;
    float* out;
    int* bad_id_flag;
} nr_kcnn_encoder_fwd_args;
int nr_kcnn_encoder_fwd(const nr_kcnn_encoder_fwd_args* a, void* stream);

typedef struct {
    long long n_seq;
    int T, d, de, F, q, n_win;
    int win[4];
    int ldx, lde, ldf, ldo, ldq;    /* ldq = round_up(q, 16)                                              */
    const long long* word_ids;
    const long long* entity_ids;
    int V, Ve;
    const void* wT_word_bf16;       /* [max x][d][n_win*ldf]: tap s' holds W_(w, max x - 1 - s')^T in columns w ldf .. w ldf + F */
    const void* wT_entity_bf16;     /* the same for the entity channel                                    */
    const void* m_bf16;             /* [de][sec] transform_matrix                                          */
    const void* wa_bf16;            /* [q][ldf]                                                           */
    const void* waT_bf16;           /* [F][ldq]                                                           */
    const float* ba;
    const float* qv;
    const void* X2_bf16;
    const void* E_bf16;
    const void* Y_bf16;
    const float* w;
    const float* dout;              /* [n_seq][ldo]                                                       */
    float* dWconv_ext;              /* [sum x_w * F][ldx] (+=); column sec + d of each window's tap 0 is d(bias) */
    float* dM_ext;                  /* [d][lde] (+=): d(transform_matrix)^T, column de = d(transform_bias)   */
    float* dWa_ext;                 /* [q][ldf] (+=); column F is d(bias)                                   */
    float* dqv;                     /* [q] (+=)                                                           */
    float* dword;                   /* [V][d] (+=)                                                        */
    float* dentity;                 /* [Ve][de] (+=)                                                      */
    void* workspace;
    long long workspace_bytes;
} nr_kcnn_encoder_bwd_args;
long long nr_kcnn_encoder_bwd_workspace(long long n_seq, int T, int d, int F, int q, int n_win);
int nr_kcnn_encoder_bwd(const nr_kcnn_encoder_bwd_args* a, void* stream);

/* ---- generic Linear over dense fp32 rows (TANR topic predictor src/model/TANR/__init__.py:58-61, GRU
 * projections).  fwd: X_bf16 = bf16(x | 1) (saved), out = act(X W^T + b).  bwd: dW_ext[N][ldx] += dY^T [X|1]
 * (column K = d(bias)), dx = dY W (optional).  relu_out masks dy with (relu_out > 0). */
int nr_linear_rows_fwd(const float* x, long long n, int K, long long s_row, long long s_col, void* X_bf16, int ldx,
                       const void* W_bf16, int N, int ldw, const float* bias, int relu, float* out, int ld_out,
                       void* stream);
int nr_linear_rows_bwd(const float* dy, const float* relu_out, long long n, int N, int ld_dy, void* dY_bf16, int ldn,
                       const void* X_bf16, int K, int ldx, const void* WT_bf16, int ldwT, float* dW_ext, float* dx,
                       int ld_dx, void* stream);

/* ---- fp32 embedding lookups (LSTUR category / user embeddings, src/model/LSTUR/news_encoder.py:47-53) ---- */
int nr_embedding_f32_fwd(const long long* ids, long long n, const float* table, int V, int D, float* out,
                         int* bad_id_flag, void* stream);
/* ids outside [1, V) contribute nothing (row 0 = padding_idx; out-of-range ids are flagged by the forward lookup) */
int nr_embedding_f32_bwd(const long long* ids, long long n, const float* dout, int V, int D, float* dtable, void* stream);

/* ---- reference: NAML ElementEncoder  relu(Linear(embedding(id)))  (src/model/NAML/news_encoder.py:40-47) --- */
int nr_element_encoder_fwd(const long long* ids, long long n, const void* table_bf16, int V, int E, int lde,
                           void* E_bf16, const void* W_bf16, int F, const float* bias, float* out, int* bad_id_flag,
                           void* stream);
int nr_element_encoder_bwd(const long long* ids, long long n, const float* dout, const float* out, int F, void* dY_bf16,
                           int ldf, const void* E_bf16, int E, int lde, const void* WT_bf16, float* dW_ext,
                           float* dtable, int V, void* stream);

/* ---- reference: LSTUR UserEncoder -- pack_padded_sequence + nn.GRU, last hidden state -----------------
 * (src/model/LSTUR/user_encoder.py:16-45).  Gate order r, z, n; user b consumes the FIRST len[b] positions of
 * its (left-padded) history (reference quirk kept as-is); len 0 is clamped to 1 (user_encoder.py:27).
 * ldd = round_up(D+1, 8), ldh = round_up(Hd+1, 8), ldg = round_up(3Hd, 4), ldb = round_up(3Hd+1, 8). */
typedef struct {
    int B, S, D, Hd;
    const float* x;                 /* fp32 [B][S][D] clicked-news vectors with element strides below     */
    long long x_s_b, x_s_t, x_s_c;
    const long long* len;           /* [B] int64 (device)                                                */
    const float* h0;                /* [B][Hd] initial hidden state (user embedding for 'ini', zeros for 'con') */
    const void* wih_bf16;           /* [3Hd][ldd]                                                        */
    const void* whh_bf16;           /* [3Hd][ldh]                                                        */
    const float* bih;
    const float* bhh;
    /* saved for backward (caller-allocated) */
    void* xb;                       /* bf16 [B*S][ldd]                                                   */
    float* gi;                      /* fp32 [B*S][ldg]   input projections, rows b*S+t                    */
    float* gh;                      /* fp32 [S][B][ldg]  recurrent projections                            */
    float* hs;                      /* fp32 [S+1][B][Hd] hidden states                                    */
    void* hb;                       /* bf16 [S+1][B][ldh]                                                 */
    float* out;                     /* fp32 [B][Hd] last hidden state                                     */
    /* accurate mode (non-NULL): the input enters the projection as a hi/lo bf16 pair, gi = x_hi.W^T + b + x_lo.W^T (two passes) */
    void* x_lo_bf16;                /* [B*S][ldd] workspace: bf16(x - bf16(x))                                         */
} nr_gru_fwd_args;
int nr_gru_fwd(const nr_gru_fwd_args* a, void* stream);
/* 1 if nr_gru_fwd runs the whole recurrence as ONE cooperative launch for this shape on this device (users in 128-row tiles x
 * hidden units in slices of 32, one CTA each, all resident): B >= 1, Hd % 4 == 0, 32 <= Hd <= 1024 (16 resident 64-column
 * k-chunks of W_hh) and ceil(B / 128) * ceil(Hd / 32) <= SM count; else it runs a GEMM, a copy and a gate kernel per step */
int nr_gru_persistent_supported(int B, int Hd);

typedef struct {
    int B, S, D, Hd;
    const long long* len;
    const void* wihT_bf16;          /* [D][ldb]  = W_ih^T                                                */
    const void* whhT_bf16;          /* [Hd][ldb] = W_hh^T                                                */
    const void* xb;
    const float* gi;
    const float* gh;
    const float* hs;
    const void* hb;
    const float* dout;              /* [B][Hd]                                                           */
    float* dWih_ext;                /* [3Hd][ldd] (+=), column D  = d(bias_ih)                            */
    float* dWhh_ext;                /* [3Hd][ldh] (+=), column Hd = d(bias_hh)                            */
    float* dx;                      /* [B*S][D] (=)                                                      */
    float* dh0;                     /* [B][Hd] (=)                                                       */
    void* workspace;
    long long workspace_bytes;
} nr_gru_bwd_args;
long long nr_gru_bwd_workspace(int B, int S, int D, int Hd);
int nr_gru_bwd(const nr_gru_bwd_args* a, void* stream);

/* ---- reference: Hi-Fi Ark after the news encoder, fp32 on the CUDA cores ---------------------------------------------------
 *   user side  SelfAttention + residual + OMAP (src/model/general/attention/self.py, src/model/HiFiArk/OMAP.py):
 *              X = hist[b] (H x F);  Y = softmax_row(X X^T) X + X;  archive[b] = softmax_over_h(Y W)^T Y  (P x F);  W is F x P
 *   scorer     SimilarityAttention + DNNClickPredictor (src/model/general/attention/similarity.py, click_predictor/DNN.py):
 *              w = softmax(A c);  u = w^T A;  logit = w2 . relu(W1 [c; u] + b1) + b2;  W1 is hidden x 2F, b2 one float
 *   regulariser (src/model/HiFiArk/OMAP.py:36-44): reg_out = || (W^T W) * (1 - I) ||_F, its gradient 2 W (M * W^T W) / R (zero at R = 0)
 * Supported bounds: 1 <= H <= 50, 4 <= F <= 400 with F % 4 == 0, 1 <= P <= 32, 1 <= hidden <= 32; a shape outside them returns -2
 * before any launch.  Shared memory per CTA: user side 4 * ((max(H, P) + H)(F + 4) + 2H^2 + 2HP + P^2 + 8) bytes (198.5 KB at the
 * bounds' corner), scorer forward 4 * (P (F + 4) + 2F + 128) bytes, scorer backward 4 * (2P (F + 4) + 2 hidden F + 4F + 260) bytes
 * (213 KB at the corner).  hist, archive and darchive must be 16-byte aligned.  The kernels have no waits, so they never write the
 * watchdog record (nr_device_error stays 0).
 * Weight gradients (dW, dW1, db1, dw2, db2) are ADDED (+=) in a fixed order: per-CTA partial rows in the workspace, summed by one
 * ordered reduction (bit-identical across runs).  dhist, dcand and darchive are written (=). */
int nr_archive_user_fwd(const float* hist, long long B, int H, int F, int P, const float* W, float* archive, float* reg_out,
                        void* stream);     /* hist [B][H][F], archive [B][P][F] (=); reg_out: device float or NULL (not computed) */
long long nr_archive_user_bwd_workspace(long long B, int F, int P);
/* dreg: device float, the gradient of reg_out, or NULL (no regulariser term) */
int nr_archive_user_bwd(const float* hist, long long B, int H, int F, int P, const float* W, const float* darchive, const float* dreg,
                        float* dhist, float* dW, void* workspace, long long workspace_bytes, void* stream);
/* Segment s (a training user, an evaluation impression) scores candidates i in [seg_offsets[s], seg_offsets[s+1]) against
 * archive[s] ([n_seg][P][F]): the candidate vector is news[cand[i]] (news [n_news][F]), or news[i] when cand is NULL.  A cand
 * index outside [0, n_news) sets *bad_id_flag and leaves NaN as its logit.  logits [n_cand] (=). */
int nr_archive_score_fwd(const float* news, long long n_news, int F, const long long* cand, long long n_cand,
                         const long long* seg_offsets, long long n_seg, const float* archive, int P, const float* W1, const float* b1,
                         int hidden, const float* w2, const float* b2, float* logits, int* bad_id_flag, void* stream);
long long nr_archive_score_bwd_workspace(long long n_seg, int F, int hidden);
/* dcand [n_cand][F] (=) by candidate POSITION i (not news row), darchive [n_seg][P][F] (=); dW1, db1, dw2, db2 (+=) */
int nr_archive_score_bwd(const float* news, long long n_news, int F, const long long* cand, long long n_cand,
                         const long long* seg_offsets, long long n_seg, const float* archive, int P, const float* W1, const float* b1,
                         int hidden, const float* w2, const float* b2, const float* dlogits, float* dcand, float* darchive,
                         float* dW1, float* db1, float* dw2, float* db2, void* workspace, long long workspace_bytes, void* stream);

/* ---- reference: DKN's history attention (src/model/DKN/attention.py), fp32 on the CUDA cores --------------------------------
 * The reference scores history row h_j against candidate c as Linear(16,1)(Linear(2F,16)([c; h_j])), with nothing between the
 * two Linears, so the score is alpha.c + beta.h_j + const with beta = W1[:, F:]^T w2: the softmax over j cancels everything
 * but beta.h_j and the user vector is the same for every candidate:
 *   user[b] = sum_j softmax_j(beta . hist[b][j]) hist[b][j]          W1 is hidden x 2F (the candidate half is never read)
 * The gradients of W1[:, :F], b1 and b2 are exactly zero; the backward adds nothing there.  One CTA per user.
 * Bounds: 1 <= H <= 64, 1 <= F <= 512, 1 <= hidden <= 32; a shape outside them returns -2 before any launch.
 * dW1 (history half) and dw2 are ADDED (+=) in a fixed order (per-CTA partial rows, one ordered reduction); dhist is written (=). */
int nr_dkn_user_fwd(const float* hist, long long B, int H, int F, const float* W1, int hidden, const float* w2, float* user,
                    void* stream);     /* hist [B][H][F], user [B][F] (=) */
long long nr_dkn_user_bwd_workspace(long long B, int F);
int nr_dkn_user_bwd(const float* hist, long long B, int H, int F, const float* W1, int hidden, const float* w2, const float* duser,
                    float* dhist, float* dW1, float* dw2, void* workspace, long long workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEWSREC_B200_H */
