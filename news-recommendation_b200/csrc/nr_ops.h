// Internal (C++) operator layer between the kernels and the C-ABI (abi.cu).  All pointers are device
// pointers, all work is enqueued on `stream`, nothing is allocated except in the debug GEMM backend.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nr {

struct DropoutCfg {
    float p;        // 0 => off
    uint64_t seed;
};

struct RowMapCfg {  // see RowMap in nr_epilogues.cuh; seg_in == 0 => identity
    int seg_in, in_off, seg_len, seg_out, out_off;
};

// ---- wgmma GEMMs with fused epilogues (gemm.cu) ------------------------------------------------
constexpr int kGemmTileRows = 64;  // rows of A per gemm_nt tile
// Operands of the GEMMs with optional epilogue features, which callers name: gemm_store({.A = X, .M = M, ...}, {.out = Y, ...}, st).
// A bf16 [M x K] pitch lda; W bf16 [taps * w_tap_rows x K] pitch ldw.  Tap s (taps <= 4) reads row r + s - tap_origin of A;
// tap_origin < 0 is the centred window taps / 2 (taps 3: the zero-padded CNN layout, tap s reads row r + s - 1)
struct GemmOperands {
    const void* A;
    int M, lda;
    const void* W;
    int N, ldw, K, taps = 1, w_tap_rows = 0, tap_origin = -1;
};

// out[M x N] = act(A . W^T + bias), bf16 or fp32; the defaults are fp32 "=", identity rows, no dropout
struct StoreCfg {
    void* out;
    int ld_out, out_bf16 = 0, relu = 0;
    int tanh = 0;  // act = tanh (fast_tanh, absolute error ~2e-7: far below the bf16 store that follows it)
    // non-null: the result is multiplied by 1 - t^2, t = dtanh_src[row][col] (bf16, pitch dtanh_ld; the output's own row and
    // column): the tanh backward through a stored bf16 activation
    const void* dtanh_src = nullptr;
    int dtanh_ld = 0;
    const float* bias = nullptr;
    RowMapCfg rm = {};
    DropoutCfg drop = {};
    int ones_col = -1, ones_zero_upto = 0;  // bf16 output: column ones_col = 1, (ones_col, ones_zero_upto) = 0 (bias of the next GEMM)
    // bf16 output, identity rows: columns [lo_col0, N) also leave a LOW plane lo[r][c - lo_col0] = bf16(y - bf16(y)) in lo_out
    // (bf16 [M][ld_lo]), so that a consumer can read y as a hi/lo bf16 pair (~16 mantissa bits)
    void* lo_out = nullptr;
    int ld_lo = 0, lo_col0 = 0;
    int accumulate = 0;                 // fp32 output only: out += A . W^T (+ bias)
    int rows_per_tile = kGemmTileRows;  // rows are computed independently: larger values are clamped to the tile
    const int* tile_list = nullptr;     // device list of the 64-row tiles to compute (GemmNTParams::tile_list); the others are not written
};
int gemm_store(const GemmOperands& g, const StoreCfg& c, cudaStream_t stream);
// whether gemm_store can emit the low plane of the columns [lo_col0, N) of an N x K product (host-only, no launch)
bool gemm_store_lo_supported(int N, int K, int lo_col0);

// additive-attention pooling: out[seg][D] = sum_r softmax_seg(tanh(X Wa^T + ba) . qv)_r X_r ; w_out[rows]
// X_lo (may be null): a second bf16 plane with X = X_hi + X_lo; the scores use X_hi, the pooled sum both planes.
int gemm_additive_pool(const void* X, int M, int lda, int D, const void* Wa, int q, int ldw, const float* ba,
                       const float* qv, int seg_len, float* out, int ldo, float* w_out, cudaStream_t stream,
                       const void* X_lo = nullptr);

// dPre = dscore * qv * (1 - tanh^2(X Wa^T + ba)) -> bf16 [M x ld_dpre]; dqv += sum_r dscore_r tanh(..)
int gemm_additive_dpre(const void* X, int M, int lda, int D, const void* Wa, int q, int ldw, const float* ba,
                       const float* qv, const float* dscore, void* dpre, int ld_dpre, float* dqv,
                       cudaStream_t stream);
// gemm_additive_dpre's shape checks (host-only, no launch): q in [1, 256], the dPre pitch, one weight slice of q x D
int additive_dpre_check(int q, int D, int ld_dpre);

// dX = dPre . Wa + w (x) dOut [* relu mask] [* dropout] -> bf16, on {.A = dPre, .N = D, .K = q, .W = Wa^T}; w and dOut
// (pitch ldo) are the pooling weights and output gradient of segments of seg_len rows
struct PoolDInputCfg {
    const float *w, *dout;
    int ldo, seg_len;
    void* dx;
    int ld_dx;
    RowMapCfg rm = {};
    int zero_pad_rows = 0;  // with a compact -> padded row map: also zero the pad rows around each segment
    DropoutCfg drop = {};
    const void* relu_src = nullptr;  // non-null: multiply by (relu_src > 0), pitch relu_ld (ReLU backward of the CNN)
    int relu_ld = 0;
};
int gemm_pool_dinput(const GemmOperands& g, const PoolDInputCfg& c, cudaStream_t stream);
// gemm_pool_dinput's shape checks (host-only, no launch): seg_len >= 1, the dOut staging cap, ld_dx % 8, the GEMM's plan
int pool_dinput_check(const GemmOperands& g, const PoolDInputCfg& c);

// dEmb[ids[row]] += A . W^T (embedding gradient of a [V x N] table; padding row 0 skipped) [* dropout of the gathered rows, pitch drop_ld]
struct ScatterEmbCfg {
    const long long* ids;
    float* demb;
    int V;
    RowMapCfg rm = {};
    DropoutCfg drop = {};
    int drop_ld = 0;
    // compact rows (LiveTokens): GEMM row r is token rows[r] (no token when negative; rm must be the identity), whose id and
    // dropout row it takes; tile_list (device, GemmNTParams::tile_list layout) replaces the scan for tiles with a live token
    const int* rows = nullptr;
    const int* tile_list = nullptr;
};
int gemm_scatter_emb(const GemmOperands& g, const ScatterEmbCfg& c, cudaStream_t stream);

// D[Ma x Nb] += A[:, :Ma]^T . B[rows + shift, b_col0 : b_col0 + Nb]   (fp32 accumulate into D, pitch ldd; Nb <= 512).
// k_list (device, GemmNTParams::tile_list layout): only the listed 64-row chunks of the rows are summed.
int gemm_tn_accumulate(const void* A, int Kr, int Ma, int lda, const void* B, int b_rows, int b_cols, int ldb,
                       int b_col0, int Nb, int b_row_shift, float* D, int ldd, cudaStream_t stream, const int* k_list = nullptr);
// Linear weight gradient: dW_ext[N][0..K] += dY^T . [X | 1] over M rows, dY pitch ld_dy, X read at row r + x_row_shift.  Column K of
// X is its ones column, so column K of dW_ext (same pitch ldx) is the bias gradient.  Launches of <= 512 columns, left to right.
int gemm_weight_grad(const void* dY, int M, int N, int ld_dy, const void* X, int K, int ldx, float* dW_ext, cudaStream_t stream,
                     int x_row_shift = 0, const int* k_list = nullptr);

// Padding titles of the news encoder's forward.  Title s is padding when its T ids are all 0 and row 0 of the bf16 table is an
// exact zero row (padding_idx=0 keeps it zero, a pretrained table may not).  Such a title's X rows are [0 .. 0, 1], so its
// Q|K|V rows are the bias rows in `qkv` below.  A 64-row tile is live when it holds a row of a title that is not padding.
// Nothing is read back to the host.
struct PaddingTitles {
    unsigned char* pad = nullptr;  // [n_seq] 1 = padding title
    int* tile_flags = nullptr;     // [ceil(n_seq * T / 64)] 1 = live tile
    int* live = nullptr;           // the live tiles in GemmNTParams::tile_list layout
    void* qkv = nullptr;           // with bqkv: bf16 [T][ld3] Q|K|V of a padding title (every row bf16(b_qkv))
    void* v_lo = nullptr;          // with bqkv: bf16 [T][sec] low plane of its V section, bf16(b - bf16(b))
    void* base = nullptr;          // the one stream-ordered allocation behind the buffers above
};
// table: the bf16 embedding table, pitch ld_table; d even, T <= 32.  Allocates on `stream`; free_padding_titles releases the
// buffers once every launch that reads them has been enqueued.
int padding_titles(const long long* ids, long long n_seq, int T, int d, const void* table, int ld_table, const float* bqkv, int sec,
                   int ld3, PaddingTitles* out, cudaStream_t stream);
void free_padding_titles(PaddingTitles& pt, cudaStream_t stream);

// Live tokens of the news encoder's backward.  Token r is live when its id is in [1, V), or when row 0 of the bf16 table is
// nonzero (then every token is).  A dead token's gathered row is [0 .. 0, 1] (gather_rows reads an out-of-range id as row 0),
// so its dQ|dK|dV row adds nothing to the embedding gradient and reaches the weight gradient only through the bias column.
// The compact order lists the live tokens in ascending token order.  A title without a live token is a padding title: the
// same verdict as padding_titles, from the same ids and table row.  Nothing is read back to the host.
struct LiveTokens {
    unsigned char* pad = nullptr;  // [n_seq] 1 = padding title (mask 0)
    uint32_t* mask = nullptr;      // [n_seq] bit t: token t of the title is live
    int* offset = nullptr;         // [n_seq + 1] exclusive scan of the masks' popcounts; offset[n_seq] = M', the live tokens
    int* index = nullptr;          // [n_seq * T] compact row -> token; -1 on the rows [M', round_up(M', 64)) below n_seq * T
    int* tiles = nullptr;          // the compact 64-row tiles 0 .. ceil(M' / 64) - 1 in GemmNTParams::tile_list layout
    void* qkv = nullptr;           // bf16 [T][ld3] Q|K|V of a padding title (every row bf16(b_qkv))
};
// table null: a token is live when its id is in [1, V) or its row of X is nonzero below column d (the same tokens, found by
// reading X; a dead token's row is [0 .. 0, 1] either way).  Also copies the live rows of X (bf16, pitch ldx) to Xc in
// compact order and writes zeros to the rows [M', round_up(M', 64)) below n_seq * T of Xc and of dqkv_c (bf16, pitch ld3),
// the rows a 64-row tile of the compact GEMMs reads past M'.  d even, T <= 32.  The buffers of `out` are carved from `buf`
// (16-byte aligned, live_tokens_bytes(n_seq, T, ld3) bytes): nothing is allocated, nothing is read back to the host.
long long live_tokens_bytes(long long n_seq, int T, int ld3);
int live_tokens(const long long* ids, long long n_seq, int T, int d, const void* table, int ld_table, int V, const float* bqkv,
                int sec, int ld3, const void* X, int ldx, void* Xc, void* dqkv_c, void* buf, long long buf_bytes, LiveTokens* out,
                cudaStream_t stream);

// ---- memory-bound companions (aux.cu) --------------------------------------------------------------
// fp32 rows -> zero-padded bf16 planes: every operand cast, dense-input conversion and hi/lo split in front of a GEMM.
// Row r = seq * T + tok (r < n_rows), column col < D: x = src[seq * s_seq + tok * s_tok + col * s_col] (element strides), plus
// pos[tok][col] when pos is set (fp32 [T][D] contiguous; the sum is formed in fp32 before the one rounding).  Columns [D, width)
// hold 0, except column D of the hi plane when ones_col (1.0: the bias of the next GEMM).  Each plane takes `width` columns
// (a multiple of 8, fewer than 2^33 columns in all the rows of a job) of 16-byte aligned rows of pitch ld_hi / ld_lo (multiples
// of 8); either plane may be null:
//   hi = bf16(x)          lo = bf16(x - bf16(x))   (hi + lo carries x to ~16 mantissa bits)
// The transpose of an fp32 [R][C] matrix is the job n_rows = C, D = R, s_seq = 1, s_col = its pitch.
struct Bf16Rows {
    const float* src;
    long long n_rows;
    int T = 1, D;
    long long s_seq, s_tok = 0, s_col = 1;
    const float* pos = nullptr;
    int width;
    void* hi = nullptr;
    int ld_hi = 0, ones_col = 0;
    void* lo = nullptr;
    int ld_lo = 0;
};
// Profiler key and grid cap (148 * blocks_per_sm blocks per job) of a conversion launch, one per kind of caller
struct Bf16Op {
    const char* name;
    int blocks_per_sm;
};
inline constexpr Bf16Op kCastPad{"cast_pad", 16}, kCastPadMany{"cast_pad_many", 4}, kRowsToBf16{"rows_to_bf16", 6},
    kRowsToBf16Hilo{"rows_to_bf16_hilo", 8}, kRowsToBf16Planes{"rows_to_bf16_planes", 8}, kRowsToBf16Lo{"rows_to_bf16_lo", 8};
// up to kBf16RowsJobs jobs in ONE launch; jobs without rows or columns are skipped, no launch when none is left
constexpr int kBf16RowsJobs = 8;
int rows_to_bf16(const Bf16Rows* jobs, int n_jobs, Bf16Op op, cudaStream_t stream);
inline int rows_to_bf16(const Bf16Rows& job, Bf16Op op, cudaStream_t stream) { return rows_to_bf16(&job, 1, op, stream); }
// dst[e] += sum_s src[s*L + e] (e < L, s < n_seq): fixed summation order, bit-identical across runs
int sum_over_seq(const float* src, long long n_seq, long long L, float* dst, cudaStream_t stream);
// X[row(seg,t)] = table_bf16[ids[seg*T+t]] (bit-exact copy), ones column at D, optional dropout, optional padded layout.
// X may be wider than the table (ld_x >= ld_table): only its first ld_table columns are written.
int gather_rows(const long long* ids, long long n_tok, int T, const void* table, int V, int D, int ld_table, void* X,
                int ld_x, int padded, DropoutCfg drop, int* bad_id_flag, cudaStream_t stream);
// the news encoder's backward over live tokens (LiveTokens above): what the title-level attention backward needs of it
struct TitleBwdLive {
    const LiveTokens* tokens;
    float* dbias;  // the bias column of the Q|K|V weight gradient
    int ld_dbias;
};
// multi-head self attention core on packed Q|K|V bf16 [n_seq*T x ld_qkv]: sections start at columns 0, sec, 2*sec
// (sec >= d = heads*dk; dQKV uses the same sections)
int mhsa_core_fwd(const void* qkv, int ld_qkv, int sec, long long n_seq, int T, int heads, int dk, void* ctx, int ld_ctx,
                  DropoutCfg drop, cudaStream_t stream);
int mhsa_core_bwd(const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int T, int heads, int dk,
                  void* dqkv, int ld_dqkv, cudaStream_t stream, const TitleBwdLive* live = nullptr);
// title-level backward (attn_title.cu): T = 20, d_k = 20, <= 15 heads, sections with a 16-byte phase (sec % 8 == 0)
bool mhsa_title_fwd_supported(int T, int dk, int heads, int sec, int ld_qkv, int ld_ctx);
// pad (PaddingTitles, may be null): the padding titles take their Q|K|V rows (and V low plane) from pad->qkv / pad->v_lo, not
// from qkv / v_lo, whose rows they may have left unwritten
int mhsa_title_fwd(const void* qkv, int ld_qkv, int sec, long long n_seq, int heads, void* ctx, int ld_ctx, DropoutCfg drop,
                   cudaStream_t stream, const void* v_lo = nullptr, int ld_vlo = 0, void* ctx_lo = nullptr,
                   const PaddingTitles* pad = nullptr);
bool mhsa_title_bwd_supported(int T, int dk, int heads, int sec, int ld_qkv, int ld_dctx, int ld_dqkv);
// live (may be null): the padding titles take their Q|K|V rows from live->tokens->qkv; only the live tokens' dQ|dK|dV rows are
// stored, in compact order (row live->tokens->offset[s] + rank of the token among its title's live tokens); the bf16-rounded
// dQ|dK|dV rows of the dead tokens are summed into dbias[c * ld_dbias] (+=), c < 3 * sec
int mhsa_title_bwd(const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int heads, void* dqkv,
                   int ld_dqkv, cudaStream_t stream, const TitleBwdLive* live = nullptr);
// dscore_r = w_r (dw_r - sum_seg w dw), dw_r = dOut[seg] . X_r
int pool_dscore(const void* X, int lda, int D, long long n_seg, int seg_len, const float* w, const float* dout, int ldo,
                float* dscore, cudaStream_t stream);
// pool_dscore's shape checks (host-only, no launch): 1 <= seg_len <= 128, D % 4, ldo % 4, lda % 8
int pool_dscore_check(int lda, int D, int seg_len, int ldo);
// logits[b][c] = cand[b][c] . user[b]
int dot_score_fwd(const float* cand, const float* user, int B, int C, int D, float* logits, cudaStream_t stream);
int dot_score_bwd(const float* cand, const float* user, const float* dlogits, int B, int C, int D, float* dcand,
                  float* duser, cudaStream_t stream);

// dst bf16 [n][ldn] = dy[n][N] (pitch ld_dy) masked by (relu_out > 0) when relu_out != null (same pitch); zero padded
int accumulate_ext_grad(float* ext, int rows, int ld, int D, float* dW, float* db, cudaStream_t stream);
int relu_bwd_to_bf16(const float* dy, const float* relu_out, long long n, int N, int ld_dy, void* dst, int ldn, cudaStream_t stream);
// fp32 embedding lookup / scatter-add (padding row 0: value read as-is, gradient skipped)
int embedding_f32_fwd(const long long* ids, long long n, const float* table, int V, int D, float* out, int* bad_id_flag,
                      cudaStream_t stream);
int embedding_f32_bwd(const long long* ids, long long n, const float* dout, int V, int D, float* dtable, cudaStream_t stream);


// ---- persistent GRU recurrence (gru_persist.cu): all S steps of h_t = GRU(gi_t, h_{t-1}) in one cooperative launch --------
int gru_persistent_supported(int B, int Hd);
int gru_fwd_persistent(int B, int S, int Hd, int ldh, int ldg, const float* gi, const void* whh, const float* bhh, const float* h0,
                       const long long* len, float* gh, float* hs, void* hb, float* out, cudaStream_t stream);
void set_gru_stepwise(int on);  // nr_debug_set_gru_stepwise (gru.cu)

// precise user encoder (NRMS precise mode): fp32 attention with hi/lo context planes
int mhsa_f32_fwd(const float* qkv, int ld, int sec, long long n_seq, int T, int heads, int dk, void* c_hi, void* c_lo, int ldc,
                 cudaStream_t stream);
// scores[i] = news[cand[i]] . user[s] for seg_offsets[s] <= i < seg_offsets[s+1]  (batched evaluate.py:245-265)
int segment_dot(const float* news, long long n_news, int D, const long long* cand, long long n_cand, const long long* seg_offsets,
                long long n_seg, const float* user, float* scores, int* bad_flag, cudaStream_t stream);
// metrics[s] = {AUC, MRR, nDCG@5, nDCG@10} of impression s (batched evaluate.py:160-168, 267-271)
int impression_metrics(const float* scores, const unsigned char* labels, const long long* seg_offsets, long long n_seg, double* metrics,
                       int* bad_label_flag, cudaStream_t stream);
// ranks[i] = place_i + 1 (the place impression_metrics uses); the prediction.txt lines of the ranks: their byte offsets (a CUB
// exclusive scan of the line lengths in the caller's workspace of prediction_scan_bytes), then every line's bytes
int impression_ranks(const float* scores, const long long* seg_offsets, long long n_seg, int* ranks, int* bad_score_flag,
                     cudaStream_t stream);
long long prediction_scan_bytes(long long n_seg);
int prediction_line_offsets(const long long* ids, const int* ranks, const long long* seg_offsets, long long n_seg, long long* line_offsets,
                            void* workspace, long long workspace_bytes, cudaStream_t stream);
int prediction_text(const long long* ids, const int* ranks, const long long* seg_offsets, long long n_seg, const long long* line_offsets,
                    char* text, cudaStream_t stream);

int slots_device_readable(const void* const* slots, int n);
int pack_slots(const void* const* slots, int H, int C, int B, int L, long long* out, cudaStream_t stream);
// one launch: every field's impression-major id block and the per-row records of a batch from the device feed's tables
// (records [R][2 + C]: user, clicked_news_length, labels -> user_out / length_out [B], clicked_out [C][B], each optional)
constexpr int kFeedFields = 8;
struct FeedField {
    const int* table;
    int width;
    long long* out;
};
struct FeedRecords {
    const int* records;
    long long *user, *length, *clicked;
};
int feed_gather(const FeedField* fields, int n_fields, const int* behaviors, int H, int C, FeedRecords rec, const long long* rows, int B,
                cudaStream_t stream);
// one launch: redraw the candidate columns [H, H + 1 + K] of the device feed's behaviour rows from each impression's
// candidates (include/newsrec_b200.h, nr_sample_negatives)
int sample_negatives(const int* cand_rows, const unsigned char* labels, const long long* imp_offsets, long long n_imp, const long long* row_offsets,
                     int K, unsigned long long seed, long long epoch, int* behaviors, int H, cudaStream_t stream);
// top-k of users . news over a whole pool, categories null, or at most max_per_category news of one category key per list
// (topk.cu; include/newsrec_b200.h, nr_topk_dot and nr_topk_dot_capped)
long long topk_dot_workspace(long long n_users, long long n_news, int D, int k);
int topk_dot(const float* users, long long n_users, int ld_users, const float* news, long long n_news, int ld_news, int D, int k,
             const long long* excl_offsets, const long long* excl_rows, const int* categories, int max_per_category, long long* idx,
             float* score, int* bad_row_flag, int* bad_score_flag, void* workspace, long long workspace_bytes, cudaStream_t stream);
// ranks of target news among a whole pool under the same scores (topk.cu; include/newsrec_b200.h, nr_pool_ranks)
long long pool_ranks_workspace(long long n_rows, long long n_news, int D);
int pool_ranks(const float* queries, long long n_rows, int ld_queries, const float* news, long long n_news, int ld_news, int D,
               const long long* tgt_offsets, const long long* tgt_rows, const long long* excl_offsets, const long long* excl_rows,
               long long* rank, float* score, int* bad_row_flag, int* bad_score_flag, int* target_flag, void* workspace,
               long long workspace_bytes, cudaStream_t stream);
int num_sms();
extern int g_launches;  // kernels launched by this library (nr_launch_count)

// ---- live per-kernel timing (bench.py): CUDA events on the launching stream around every kernel ------
// Off by default.  A ProfScope brackets one kernel launch; names are "<context>/<op>[shape]".
void prof_enable(int on);
void prof_context(const char* ctx);  // prefix set by the composites ("news.fwd", "user.bwd", ...)
int prof_report(char* buf, int cap); // JSON {"name": [launches, total_ms], ...}; clears the records
struct ProfScope {
    ProfScope(const char* op, int a, int b, int c, cudaStream_t s);
    ~ProfScope();
    int idx;
    cudaStream_t stream;
};

// ---- host conventions of the C-ABI composites (abi.cu, abi_cnn.cu, gru.cu) --------------------------
static inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }
static inline long long align256(long long x) { return (x + 255) & ~255ll; }
// Dropout on the attention context / conv output: the forward and the backward of a composite must draw this same mask.
// The Python reference model of the kernels (the oracle) restates the salt for the same two masks.
static inline DropoutCfg context_dropout(float p, uint64_t seed) { return {p, seed ^ 0x5bd1e995u}; }
// Back-to-back 256-byte aligned slots of a backward's workspace, plus 256 bytes at the end.  Over a null base it only
// measures, so a composite's *_workspace() size and the buffers its backward carves come from one layout (derive from it).
struct WorkspaceLayout {
    char* base;
    long long used = 0;
    template <class T> T* take(long long count) {
        T* p = base != nullptr ? reinterpret_cast<T*>(base + used) : nullptr;
        used += align256(count * static_cast<long long>(sizeof(T)));
        return p;
    }
    long long bytes() const { return used + 256; }
};

}  // namespace nr
