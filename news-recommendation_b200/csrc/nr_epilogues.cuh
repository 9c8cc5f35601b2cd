// Fused epilogue functors for gemm_nt.  A tile (64 rows) belongs to one consumer warpgroup, 128 threads.  A fragment-view
// functor (kFragmentView, EpiStore) gets frag(acc, FragCtx): warp w of the warpgroup handles tile rows 16w .. 16w + 15 of every
// column of the slice straight from the wgmma fragment.  A row-view functor gets operator()(acc, EpiCtx): thread t of the
// warpgroup owns accumulator row r = 32*((t>>5)&1) + lane and column half t>>6; the two halves split the slice's 32-column
// chunks as epi_chunk_range does ([ch0, ch1), warp-uniform).  Contract for every functor:
//   * row view: the accumulator is read through epi_chunks() (nr_gemm.cuh): c.rounds loads per tile, collective over the
//     warpgroup, acc.release() exactly once per tile
//   * operator() synchronises only its own warpgroup (epi_bar_sync(c.wg)); the other warpgroup is issuing wgmmas meanwhile
//   * init()/finish() bracket the CTA's whole tile loop (all 256 consumer threads call them; consumers_bar_sync())
//   * kScratchBytes of shared memory belong to the functor (the planner sizes the A ring around it); per-tile state is
//     kept per warpgroup
//   * per-slice vectors (bias, query vector, dOut rows) are staged in shared memory: with ~220 KB of smem carved out
//     the L1 holds next to nothing and per-element global loads made the epilogue 10x the MMA time.
//     Anything that must come from global memory per tile is fetched with many loads in flight or prefetched one
//     tile ahead with cp.async -- a dependent L2 round trip (~600 cycles) per chunk was the whole epilogue time.
#pragma once
#include "nr_gemm.cuh"

namespace nr {

// Row re-mapping between the compact token layout (segment s, token t -> row s*T + t) and the
// zero-padded CNN layout (row s*(T+2) + 1 + t; rows 0 and T+1 of every segment are zero).
struct RowMap {
    int seg_in;   // 0 => identity
    int in_off;
    int seg_len;
    int seg_out;
    int out_off;
    __device__ __forceinline__ bool map(int grow, long long& orow, int& t_out) const {
        if (seg_in == 0) { orow = grow; t_out = 0; return true; }
        const int s = grow / seg_in;
        const int t = grow - s * seg_in - in_off;
        t_out = t;
        orow = static_cast<long long>(s) * seg_out + t + out_off;
        return t >= 0 && t < seg_len;
    }
};

__device__ __forceinline__ void zero_row_bf16(__nv_bfloat16* row, int ld) {  // ld % 8 == 0, 16B aligned
    for (int i = 0; i < ld; i += 8) *reinterpret_cast<uint4*>(row + i) = make_uint4(0u, 0u, 0u, 0u);
}

// SWIZZLE_64B layout of a tile with 64-byte rows (32 bf16): byte offset of 16-byte piece q of row r.  Eight consecutive
// rows at the same q (the rows of one stmatrix matrix, or a row-per-lane 16-byte access) land in eight different bank groups.
__device__ __forceinline__ int sw64_offset(int r, int q) { return r * 64 + ((q ^ (r >> 1)) & 3) * 16; }

// A 32-column chunk of a fragment-view epilogue's output as bf16 pairs: w[2jj + e] holds row e of the lane, columns
// 8jj + 2 (lane % 4) + {0, 1} of the chunk (the wgmma fragment's order).
// Predicated stores straight from the fragment: row e goes to output row row[e] when ok[e], chunk column c to column col + c,
// exactly the columns c < lim.
__device__ __forceinline__ void store_frag_bf16(__nv_bfloat16* out, int ld, const long long* row, const bool* ok, int col, int lim,
                                                const uint32_t* w) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int c = 8 * jj + 2 * (lane & 3);
            if (!ok[e] || c >= lim) continue;
            __nv_bfloat16* o = out + row[e] * ld + col + c;
            if (c + 1 < lim) *reinterpret_cast<uint32_t*>(o) = w[2 * jj + e];
            else *o = __ushort_as_bfloat16(static_cast<unsigned short>(w[2 * jj + e]));  // the pair's low half: column c
        }
}

// The staging boxes of a fragment-view epilogue, built per tile by every lane of a consumer warp.  Each warp owns a ring of
// kBoxes boxes of 16 rows x 32 bf16 (its rows of one chunk) in the SWIZZLE_64B layout; a chunk is packed into the next box
// with two stmatrix and leaves by one lane's TMA store (send: rows >= M and columns past the map are clipped by the map) or
// as 16-byte row pieces to mapped rows (put_rows).  With TMA the ring lets kBoxes - 1 of the warp's stores be in flight while
// a box is written; the CTA's last ones are drained by finish().
template <int kBoxes>
struct FragStore {
    static constexpr int kBoxBytes = 16 * 64;
    static constexpr int kScratchBytes = kEpiWarps * kBoxes * kBoxBytes + 1024;  // + alignment slack
    uint32_t ring;       // this warp's first box
    uint32_t st_off[2];  // stmatrix x of a chunk writes the 8 x 8 matrices (jj, e) = (2x + m/2, m%2), m = lane / 8
    int row;             // global row of the boxes' row 0
    int tma;
    int n = 0;           // chunks staged in this tile

    // scratch: where the epilogue's boxes begin (aligned up to 1 KB here)
    __device__ __forceinline__ FragStore(const float* scratch, const FragCtx& f, int use_tma)
        : row(f.row0 + 16 * f.wq), tma(use_tma) {
        const int lane = threadIdx.x & 31;
        ring = ((smem_u32(scratch) + 1023u) & ~1023u) + (threadIdx.x >> 5) * (kBoxes * kBoxBytes);
#pragma unroll
        for (int x = 0; x < 2; ++x) {
            const int m = lane >> 3;
            st_off[x] = sw64_offset(8 * (m & 1) + (lane & 7), 2 * x + (m >> 1));
        }
        if (tma) {  // the previous tile's stores have left the boxes (the other warpgroup's MMAs ran in between)
            if (lane == 0) bulk_wait_read<0>();
            __syncwarp();
        }
    }
    __device__ __forceinline__ uint32_t stage(const uint32_t* w) {
        const uint32_t box = ring + (n % kBoxes) * kBoxBytes;
        if (tma && n >= kBoxes) {  // the store issued from this box kBoxes stores ago has been read out
            if ((threadIdx.x & 31) == 0) bulk_wait_read<kBoxes - 1>();
            __syncwarp();
        }
        stmatrix_x4(box + st_off[0], w[0], w[1], w[2], w[3]);
        stmatrix_x4(box + st_off[1], w[4], w[5], w[6], w[7]);
        ++n;
        return box;
    }
    __device__ __forceinline__ void send(const CUtensorMap* tm, const uint32_t* w, int col) {
        const uint32_t box = stage(w);
        fence_proxy_async();
        __syncwarp();
        if ((threadIdx.x & 31) == 0) {
            tma_store_2d(tm, box, col, row);
            bulk_commit();
        }
    }
    // row r of the box leaves as 4 x 16 bytes to output row orow[r / 8] (when v[r / 8]), lane = 4 (r % 8) + piece: each lane
    // writes its own rows.  The next put_rows' __syncwarp orders these reads before the box is written again (kBoxes >= 2).
    __device__ __forceinline__ void put_rows(__nv_bfloat16* out, int ld, const long long* orow, const bool* v, const uint32_t* w,
                                             int col) {
        const int lane = threadIdx.x & 31;
        const uint32_t box = stage(w);
        __syncwarp();
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int q = lane & 3;
            const uint4 u = lds_u4(box + sw64_offset((lane >> 2) + 8 * e, q));
            if (v[e]) *(reinterpret_cast<uint4*>(out + orow[e] * ld + col) + q) = u;
        }
    }
    // end of the CTA's tile loop (every consumer thread)
    static __device__ __forceinline__ void finish(const EpiInit& e) {
        if ((e.tid & 31) == 0) bulk_wait_all();
    }
};

// The dOut rows a pool-backward tile reads, staged per warpgroup in shared memory: every segment the 64-row tile touches
// (<= 64/seg_len + 2), slice columns only, [segment][pitch round_up(ncols, 4)] so that every staged row is 16-byte aligned.
// Two buffers of kStageFloats per warpgroup: the one of the warpgroup's NEXT tile is filled by cp.async while this one is read.
struct DOutStage {
    static constexpr int kStageFloats = 1536;
    static constexpr int kScratchBytes = 4 * kStageFloats * 4;
    const float* dout;  // [segments][ldo]
    int ldo;
    int seg_len;
    int M;

    static __device__ __forceinline__ int pitch(int ncols) { return (ncols + 3) & ~3; }
    // the 128 threads of a warpgroup (wtid): queue the dOut rows of `tile` (columns [col0, col0 + ncols)) into buf
    __device__ __forceinline__ void stage_tile(int tile, int col0, int ncols, int wtid, float* buf) const {
        const int row0 = tile * kTileM, sp = pitch(ncols);
        const int seg_first = row0 / seg_len;
        const int seg_last = min(row0 + kTileM - 1, M - 1) / seg_len;
        const int total = (seg_last - seg_first + 1) * sp;
        for (int i = wtid; i < total; i += kWgThreads) {
            const int sgi = i / sp, j = i - sgi * sp;
            const bool ok = j < ncols;
            cp_async_f32(buf + i, dout + static_cast<size_t>(seg_first + sgi) * ldo + (ok ? col0 + j : 0), ok);
        }
        cp_async_commit();
    }
    __device__ __forceinline__ void init(const EpiInit& e, int tile_step) const {  // each warpgroup queues its own first tile
        const int wg = e.tid >> 7, first = e.first_tile + wg * tile_step;
        if (first < e.num_tiles) stage_tile(first, e.col0, e.ncols, e.tid & 127, e.scratch + 2 * wg * kStageFloats);
    }
    // per tile, the whole warpgroup: wait for this tile's rows and queue the next tile's; returns this tile's buffer
    __device__ __forceinline__ const float* begin(float* scratch, int wg, int it, int next_tile, int col0, int ncols) const {
        float* mine = scratch + 2 * wg * kStageFloats;
        cp_async_wait_all();
        epi_bar_sync(wg);  // this tile's dOut rows are visible; the warpgroup is done with its other buffer
        if (next_tile >= 0) stage_tile(next_tile, col0, ncols, threadIdx.x & 127, mine + ((it + 1) & 1) * kStageFloats);
        return mine + (it & 1) * kStageFloats;
    }
    // the staged dOut row of global row grow, in the tile whose first row is row0 (the first staged row when !valid)
    __device__ __forceinline__ const float* row(const float* buf, int row0, int grow, bool valid, int ncols) const {
        return buf + (valid ? grow / seg_len - row0 / seg_len : 0) * pitch(ncols);
    }
};

__device__ __forceinline__ bool aligned32(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31) == 0; }

__device__ __forceinline__ void store_bf16x8(__nv_bfloat16* o, const float* y, int nvalid) {
    if (nvalid == 8) {
        *reinterpret_cast<uint4*>(o) =
            make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7]));
    } else {  // fully unrolled + predicated: a run-time index into y would push the caller's accumulator registers to local memory
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < nvalid) o[j] = __float2bfloat16_rn(y[j]);
    }
}

// ------------------------------------------------------------------------------------------------
// out = act(acc + bias) [* dropout]  ->  bf16 or fp32, optional row re-map, optional "ones" column, optional low plane
// Fragment view: every output element is independent, so each warp writes its own 16 rows of the tile straight from the
// wgmma fragment, with no transpose and no barrier across warps.  A 32-column bf16 chunk is packed into one of the warp's
// staging boxes with stmatrix and leaves by TMA (identity rows) or as 16-byte row pieces (mapped rows); fp32 output and bf16
// chunks cut by the slice's end leave from the fragment, a quad of lanes covering 8 contiguous columns of a row.
// scratch: [0, 1 KB) bias of the slice (zero past ncols) | the staging boxes (FragStore, 1 KB aligned)
// ------------------------------------------------------------------------------------------------
struct EpiStore {
    static constexpr bool kFragmentView = true;
    // a slice issues up to 2 x 8 stores per tile; the ring lets six of them be in flight before a box is reused
    using Store = FragStore<6>;
    static constexpr int kScratchBytes = 1024 + Store::kScratchBytes;
    CUtensorMap tm_out;  // bf16 output as a TMA tensor (32 x 16 boxes, SWIZZLE_64B); valid when use_tma
    CUtensorMap tm_lo;   // low plane of the columns >= lo_col0 (bf16(y - bf16(y))), its column 0 = output column lo_col0
    int accumulate;      // fp32 output only: out += result
    int lo_col0;         // < 0: no low plane
    __nv_bfloat16* lo_out;  // the same plane for the chunks that leave without TMA; pitch ld_lo
    int ld_lo;
    int use_tma;         // identity row map + bf16 output + whole 64-row tiles: bf16 chunks leave through tm_out / tm_lo
    void* out;
    int ld;
    int out_bf16;
    const float* bias;  // may be null
    int relu;
    int act_tanh;       // y = tanh(acc + bias)
    const __nv_bfloat16* dtanh_src;  // non-null: y *= 1 - t^2, t = dtanh_src[output row][output column] (pitch dtanh_ld)
    int dtanh_ld;
    int N;              // total valid columns
    RowMap rm;
    Dropout drop;
    int ones_col;       // >=0: column set to 1.0 (bias-gradient trick for the next weight-grad GEMM); -1 off
    int ones_cols_zero_upto;  // columns (ones_col, upto) are zeroed
    int dbg_skip;       // tuning only (NEWSREC_EPI_DBG=1): leave the accumulators untouched -> MMA/TMA pipeline alone

    __device__ void init(const EpiInit& e, int) const {
        for (int i = e.tid; i < 256; i += kEpiThreads) e.scratch[i] = (bias != nullptr && i < e.ncols) ? bias[e.col0 + i] : 0.f;
        consumers_bar_sync();
    }
    __device__ void finish(const EpiInit& e) const {
        if (use_tma) Store::finish(e);
    }

    __device__ __forceinline__ void frag(const float* acc, const FragCtx& f) const {
#ifdef NEWSREC_TRIAGE
        if (dbg_skip) return;
#endif
        const int lane = threadIdx.x & 31;
        // this lane's rows e = 0, 1: tile row 16 wq + lane / 4 + 8e
        long long orow[2];
        bool v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int r = 16 * f.wq + (lane >> 2) + 8 * e;
            int t;
            v[e] = rm.map(f.row0 + r, orow[e], t) && r < f.rows;
        }
        Store st(f.scratch + 256, f, use_tma);
        // a bf16 chunk of 32 output columns from column col: a chunk cut by the slice's end leaves from the fragment with
        // predicated stores, which write exactly the columns < ncols (letting the tensor map clip it at N changed the outputs
        // where N % 16 != 0)
        auto put = [&](__nv_bfloat16* base, int ldo, const CUtensorMap* tm, const uint32_t* w, int lc0, int col) {
            if (lc0 + 32 > f.ncols) store_frag_bf16(base, ldo, orow, v, col, f.ncols - lc0, w);  // warp-uniform
            else if (use_tma) st.send(tm, w, col);
            else st.put_rows(base, ldo, orow, v, w, col);
        };
        auto put_f32 = [&](const float* y, int lc0) {  // y[4jj + 2e + i]: row e, slice column lc0 + 8jj + 2 (lane % 4) + i
#pragma unroll
            for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int lc = lc0 + 8 * jj + 2 * (lane & 3);
                    if (!v[e] || lc >= f.ncols) continue;
                    const float y0 = y[4 * jj + 2 * e], y1 = y[4 * jj + 2 * e + 1];
                    float* o = static_cast<float*>(out) + orow[e] * ld + f.col0 + lc;
                    if (lc + 1 < f.ncols) {
                        float2 r = make_float2(y0, y1);
                        if (accumulate) {  // out += : second pass of a split-operand product (x_lo . W^T on top of x_hi . W^T)
                            const float2 o2 = *reinterpret_cast<const float2*>(o);
                            r.x += o2.x; r.y += o2.y;
                        }
                        *reinterpret_cast<float2*>(o) = r;
                    } else {
                        *o = accumulate ? *o + y0 : y0;
                    }
                }
        };
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            if (q < f.nch) {  // a compile-time chunk index keeps the fragment in registers
                const int lc0 = 32 * q;
                float y[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) y[k] = acc[16 * q + k];
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {  // bias from shared memory (zero past ncols)
                    const float2 b = lds_f2(f.scratch + lc0 + 8 * jj + 2 * (lane & 3));
                    y[4 * jj] += b.x; y[4 * jj + 1] += b.y; y[4 * jj + 2] += b.x; y[4 * jj + 3] += b.y;
                }
                if (relu) {
#pragma unroll
                    for (int k = 0; k < 16; ++k) y[k] = fmaxf(y[k], 0.f);
                }
                if (act_tanh) {
#pragma unroll
                    for (int k = 0; k < 16; ++k) y[k] = fast_tanh(y[k]);
                }
                if (dtanh_src != nullptr) {
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int lc = lc0 + 8 * jj + 2 * (lane & 3);
                            if (!v[e] || lc >= f.ncols) continue;
                            const float2 t = unpack_bf16x2(
                                __ldg(reinterpret_cast<const unsigned*>(dtanh_src + orow[e] * dtanh_ld + f.col0 + lc)));
                            y[4 * jj + 2 * e] *= 1.f - t.x * t.x;
                            y[4 * jj + 2 * e + 1] *= 1.f - t.y * t.y;
                        }
                }
                if (drop.active()) drop.apply_frag(y, orow, ld, f.col0 + lc0);
                if (out_bf16) {
                    const int col = f.col0 + lc0;
                    uint32_t w[8];
#pragma unroll
                    for (int k = 0; k < 8; ++k) w[k] = pack_bf16x2(y[2 * k], y[2 * k + 1]);
                    put(static_cast<__nv_bfloat16*>(out), ld, &tm_out, w, lc0, col);
                    if (lo_col0 >= 0 && col >= lo_col0) {  // warp-uniform (the host checked the chunk alignment)
#pragma unroll
                        for (int k = 0; k < 8; ++k) {
                            const float2 h = unpack_bf16x2(w[k]);
                            w[k] = pack_bf16x2(y[2 * k] - h.x, y[2 * k + 1] - h.y);
                        }
                        put(lo_out, ld_lo, &tm_lo, w, lc0, col - lo_col0);
                    }
                } else {
                    put_f32(y, lc0);
                }
            }
        }
        if (ones_col >= 0 && out_bf16 && f.col0 == 0 && (lane & 3) == 0) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (!v[e]) continue;
                __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out) + orow[e] * ld;
                o[ones_col] = __float2bfloat16_rn(1.0f);
                for (int j = ones_col + 1; j < ones_cols_zero_upto; ++j) o[j] = __float2bfloat16_rn(0.f);
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// Additive-attention pooling (reference additive.py:35-53) fused behind  pre = X.Wa^T:
//   score_r = sum_c tanh(pre_rc + ba_c) * qv_c ; w = softmax over the segment ; out_s = sum_r w_r X_r
// Requires n_slices == 1 and rows_per_tile = (segments per tile) * seg_len, seg_len <= 64.
// scratch floats: [0,256) bias | [256,512) query | per warpgroup w at 512 + 192w: [0,128) partial scores (half*64 + row),
// [128,192) softmax weights
// ------------------------------------------------------------------------------------------------
struct EpiPool {
    static constexpr int kScratchBytes = 4096;
    const float* bias;
    const float* qv;
    const __nv_bfloat16* X;  // the GEMM's A operand (rows x lda), re-read (L2 hits) for the weighted sum
    const __nv_bfloat16* X_lo;  // optional second plane (same pitch): the pooled rows are X + X_lo (hi/lo bf16 pair)
    int lda;
    int D;        // pooled width (even)
    int seg_len;
    int rows_per_tile;
    int M;
    float* out;   // [segments][ldo] fp32
    int ldo;
    float* w_out; // [rows] fp32 softmax weights (saved for backward); may be null

    __device__ void init(const EpiInit& e, int) const {
        for (int i = e.tid; i < 256; i += kEpiThreads) {
            e.scratch[i] = i < e.ncols ? bias[e.col0 + i] : 0.f;
            e.scratch[256 + i] = i < e.ncols ? qv[e.col0 + i] : 0.f;
        }
        consumers_bar_sync();
    }
    __device__ void finish(const EpiInit&) const {}

    // 16-byte column chunk ck of the rows [r0, r0 + seg_len): weighted sum with the weights in s_w, U loads in flight
    template <int U>
    __device__ __forceinline__ void wsum_rows(const uint4* xp, size_t pitch16, const float* s_w, int& t, float* a) const {
        for (; t + U <= seg_len; t += U) {
            uint4 u[U];
#pragma unroll
            for (int k = 0; k < U; ++k) u[k] = __ldg(xp + static_cast<size_t>(t + k) * pitch16);
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const float wt = lds_f(s_w + t + k);
                const uint32_t uw[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = unpack_bf16x2(uw[j]);
                    a[2 * j] = fmaf(wt, f.x, a[2 * j]);
                    a[2 * j + 1] = fmaf(wt, f.y, a[2 * j + 1]);
                }
            }
        }
    }

    template <class Acc>
    __device__ __forceinline__ void operator()(const Acc& acc, const EpiCtx& c) const {
        float score = 0.f;
        epi_chunks(
            acc, c, [](int) {},
            [&](int ch, float* x) {
                const float* sb = c.scratch + ch * 32;
                const float* sq = c.scratch + 256 + ch * 32;
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const float4 b4 = lds_f4(sb + j);
                    const float4 q4 = lds_f4(sq + j);  // zero beyond ncols: no contribution
                    score = fmaf(fast_tanh(x[j] + b4.x), q4.x, score);
                    score = fmaf(fast_tanh(x[j + 1] + b4.y), q4.y, score);
                    score = fmaf(fast_tanh(x[j + 2] + b4.z), q4.z, score);
                    score = fmaf(fast_tanh(x[j + 3] + b4.w), q4.w, score);
                }
            });
        float* s_part = c.scratch + 512 + 192 * c.wg;
        float* s_w = s_part + 128;
        static_assert(kEpiHalves == 2 && (512 + 2 * 192) * 4 <= kScratchBytes, "EpiPool scratch layout");
        auto row_score = [&](int r) { return s_part[r] + s_part[kTileM + r]; };
        s_part[c.half * kTileM + c.r] = score;
        epi_bar_sync(c.wg);
        if (c.half == 0) {
            float w = 0.f;
            if (c.valid) {
                const int s0 = (c.r / seg_len) * seg_len;
                const float mine = row_score(c.r);
                float m = -INFINITY;
                for (int t = 0; t < seg_len; ++t) m = fmaxf(m, row_score(s0 + t));
                float sum = 0.f;
                for (int t = 0; t < seg_len; ++t) sum += __expf(row_score(s0 + t) - m);
                w = __fdividef(__expf(mine - m), sum);
                if (w_out != nullptr) w_out[c.grow] = w;
            }
            s_w[c.r] = w;
        }
        epi_bar_sync(c.wg);
        // out[segment] = sum_t w_t X_t: work item = (segment, 16-byte column chunk); the rows come back from L2 and
        // the loop keeps 10 (then 4, then 1) independent loads in flight per thread.
        const int row0 = c.tile * rows_per_tile;
        const int nseg = rows_per_tile / seg_len;
        const int nck = (D + 7) >> 3;  // the A pitch is a multiple of 8 elements: the last chunk stays in bounds
        const size_t pitch16 = static_cast<size_t>(lda) >> 3;
        for (int item = c.wtid; item < nseg * nck; item += kWgThreads) {
            const int s = item / nck, ck = item - s * nck;
            const int r0 = row0 + s * seg_len;
            if (r0 >= M) continue;
            const uint4* xp = reinterpret_cast<const uint4*>(X + static_cast<size_t>(r0) * lda) + ck;
            const float* sw = s_w + s * seg_len;
            float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            int t = 0;
            wsum_rows<10>(xp, pitch16, sw, t, a);
            wsum_rows<4>(xp, pitch16, sw, t, a);
            wsum_rows<1>(xp, pitch16, sw, t, a);
            if (X_lo != nullptr) {  // low plane of a hi/lo pair: same weights, same accumulators
                const uint4* xl = reinterpret_cast<const uint4*>(X_lo + static_cast<size_t>(r0) * lda) + ck;
                t = 0;
                wsum_rows<10>(xl, pitch16, sw, t, a);
                wsum_rows<4>(xl, pitch16, sw, t, a);
                wsum_rows<1>(xl, pitch16, sw, t, a);
            }
            float* o = out + static_cast<size_t>(r0 / seg_len) * ldo + ck * 8;
            if (ck * 8 + 8 <= D && (ldo & 3) == 0) {
                *reinterpret_cast<float4*>(o) = make_float4(a[0], a[1], a[2], a[3]);
                *reinterpret_cast<float4*>(o + 4) = make_float4(a[4], a[5], a[6], a[7]);
            } else {
                for (int j = 0; j < 8 && ck * 8 + j < D; ++j) o[j] = a[j];
            }
        }
        epi_bar_sync(c.wg);  // s_w is rewritten by this warpgroup's next tile
    }
};

// ------------------------------------------------------------------------------------------------
// Backward of the additive scorer, fused behind the recomputed pre = X.Wa^T:
//   T = tanh(pre + ba);  dPre_rc = dscore_r * qv_c * (1 - T^2)  -> bf16;   dqv_c += sum_r dscore_r * T_rc
// Fragment view: every dPre element depends on its own row and column only, so each warp works on its 16 rows of the tile
// straight from the wgmma fragment (the row view's shared-memory transpose was most of this GEMM's time).  A 32-column
// chunk of dPre is packed into one of the warp's staging boxes with stmatrix and leaves by TMA; the dqv column sums of the
// chunk are reduced over the warp's rows with a 7-shuffle butterfly and added to shared memory, one column per lane.
// The output tensor map spans the whole pitch ld: the columns in [ncols, ld) are written as exact zeros (bias and query
// vector are zero there), so GEMMs that read dPre with K = ld see zero padding.
// scratch floats: [0,256) column sums | [256,512) bias | [512,768) query vector | the staging boxes (FragStore)
// ------------------------------------------------------------------------------------------------
struct EpiDPre {
    static constexpr bool kFragmentView = true;
    using Store = FragStore<4>;  // a smaller ring than EpiStore's keeps six A stages beside a 224 x 320 weight slice
    static constexpr int kScratchBytes = 3072 + Store::kScratchBytes;
    CUtensorMap tm_out;       // dpre as a TMA tensor ([rows][ld], 32 x 16 boxes, SWIZZLE_64B); valid when use_tma
    int use_tma;
    const float* bias;
    const float* qv;
    const float* dscore;      // [rows]
    __nv_bfloat16* dpre;      // [rows][ld]
    int ld;
    float* dqv;               // [q] fp32, accumulated

    __device__ void init(const EpiInit& e, int) const {
        for (int i = e.tid; i < 256; i += kEpiThreads) {
            e.scratch[i] = 0.f;
            e.scratch[256 + i] = i < e.ncols ? bias[e.col0 + i] : 0.f;
            e.scratch[512 + i] = i < e.ncols ? qv[e.col0 + i] : 0.f;
        }
        consumers_bar_sync();
    }
    __device__ void finish(const EpiInit& e) const {
        consumers_bar_sync();  // both warpgroups' column sums are in; one add per column and CTA
        for (int i = e.tid; i < e.ncols; i += kEpiThreads) atomicAdd(dqv + e.col0 + i, e.scratch[i]);
        if (use_tma) Store::finish(e);
    }

    __device__ __forceinline__ void frag(const float* acc, const FragCtx& f) const {
        const int lane = threadIdx.x & 31;
        // this lane's rows e = 0, 1: tile row 16 wq + lane / 4 + 8e (rows past the tile's end carry ds = 0: dPre = 0 there, and
        // the tensor map clips them at the last row)
        float ds[2];
        long long grow[2];
        bool v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int r = 16 * f.wq + (lane >> 2) + 8 * e;
            grow[e] = static_cast<long long>(f.row0) + r;
            v[e] = r < f.rows;
            ds[e] = v[e] ? __ldg(dscore + grow[e]) : 0.f;
        }
        Store st(f.scratch + 768, f, use_tma);
        const int b2 = (lane >> 2) & 1, b3 = (lane >> 3) & 1, b4 = (lane >> 4) & 1;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            if (q < f.nch) {  // a compile-time chunk index keeps the fragment in registers
                const int lc0 = 32 * q;
                uint32_t w[8];   // bf16 pair k: fragment group jj = k / 2, row e = k % 2
                float s[8];      // ds * T summed over the lane's two rows: s[2 jj + i] = column 8 jj + 2 (lane % 4) + i
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int lc = lc0 + 8 * jj + 2 * (lane & 3);
                    const float2 b = lds_f2(f.scratch + 256 + lc), qq = lds_f2(f.scratch + 512 + lc);
                    float t[2][2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        t[e][0] = tanh_approx(acc[16 * q + 4 * jj + 2 * e] + b.x);
                        t[e][1] = tanh_approx(acc[16 * q + 4 * jj + 2 * e + 1] + b.y);
                        w[2 * jj + e] = pack_bf16x2((ds[e] * qq.x) * fmaf(-t[e][0], t[e][0], 1.f), (ds[e] * qq.y) * fmaf(-t[e][1], t[e][1], 1.f));
                    }
                    s[2 * jj] = fmaf(ds[0], t[0][0], ds[1] * t[1][0]);
                    s[2 * jj + 1] = fmaf(ds[0], t[0][1], ds[1] * t[1][1]);
                }
                if (use_tma) st.send(&tm_out, w, f.col0 + lc0);  // columns >= ld are clipped by the map
                else store_frag_bf16(dpre, ld, grow, v, f.col0 + lc0, ld - f.col0 - lc0, w);  // even: a pair never straddles ld
                // column sums over the warp's 16 rows: reduce-scatter across lane bits 4, 3, 2 (the lanes holding the same
                // columns); lane ends with the sum of column 8 (2 b4 + b3) + 2 (lane % 4) + b2
                float s1[4], s2[2];
#pragma unroll
                for (int k = 0; k < 4; ++k) s1[k] = (b4 ? s[k + 4] : s[k]) + __shfl_xor_sync(0xffffffffu, b4 ? s[k] : s[k + 4], 16);
#pragma unroll
                for (int k = 0; k < 2; ++k) s2[k] = (b3 ? s1[k + 2] : s1[k]) + __shfl_xor_sync(0xffffffffu, b3 ? s1[k] : s1[k + 2], 8);
                const float s3 = (b2 ? s2[1] : s2[0]) + __shfl_xor_sync(0xffffffffu, b2 ? s2[0] : s2[1], 4);
                atomicAdd(f.scratch + lc0 + 8 * (2 * b4 + b3) + 2 * (lane & 3) + b2, s3);  // zero past ncols: never added to dqv
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// dX_rc = acc_rc + w_r * dOut[seg(r)][c]  (pool backward, both paths into X) [* relu mask] [* dropout] -> bf16
// Row view, for a row-mapped destination and/or a ReLU mask (the CNN encoders); the identity / no-mask case is EpiDPoolInFrag.
// scratch: the dOut rows (DOutStage) | kTileStoreBufs staging tiles per consumer warp (1 KB aligned)
// ------------------------------------------------------------------------------------------------
struct EpiDPoolIn {
    static constexpr int kScratchBytes = DOutStage::kScratchBytes + kTileStoreBytes;
    const float* w;      // [rows]
    const float* dout;   // [segments][ldo]
    int ldo;
    int seg_len;
    __nv_bfloat16* dx;   // [rows(mapped)][ld]
    int ld;
    int N;
    RowMap rm;
    int zero_pad_rows;
    Dropout drop;
    const __nv_bfloat16* relu_src;  // non-null: multiply by (relu_src[r][c] > 0) (ReLU backward of the CNN); pitch relu_ld
    int relu_ld;
    int M;

    __device__ void init(const EpiInit& e, int tile_step) const { DOutStage{dout, ldo, seg_len, M}.init(e, tile_step); }
    __device__ void finish(const EpiInit&) const {}

    template <class Acc>
    __device__ __forceinline__ void operator()(const Acc& acc, const EpiCtx& c) const {
        long long orow;
        int t;
        const bool v = rm.map(c.grow, orow, t) && c.valid;
        const float wr = c.valid ? __ldg(w + c.grow) : 0.f;
        const DOutStage dst{dout, ldo, seg_len, M};
        const float* sd = dst.row(dst.begin(c.scratch, c.wg, c.it, c.next_tile, c.col0, c.ncols), c.grow - c.r, c.grow, c.valid, c.ncols);
        const int lane = c.tid & 31;
        epi_chunks(
            acc, c, [](int) {},
            [&](int ch, float* x) {
                // a full 32-column chunk goes through the warp's two staging tiles so that the mask rows are LOADED and the
                // result rows STORED as 8 rows x 64 contiguous bytes per instruction (row-per-lane 16-byte accesses touch 32
                // half-used sectors per instruction and queue in the LSU: this epilogue ran at 0.64 ms against 0.26 ms for the
                // identity/TMA form of the same GEMM on a B200).
                const int col = c.col0 + ch * 32;
                const bool coop = ch * 32 + 32 <= c.ncols && col + 32 <= N && (col & 7) == 0 && (ld & 7) == 0 &&
                                  (relu_src == nullptr || (relu_ld & 7) == 0);  // warp-uniform
                if (coop) {
                    uint8_t* stage = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(c.scratch + DOutStage::kScratchBytes / 4) + 1023) &
                                                                ~uintptr_t(1023)) +
                                     (c.tid >> 5) * (kTileStoreBufs * 2048);
                    uint8_t* rb = stage;          // mask tile  (32 rows x 64 bytes, SWIZZLE_64B like WarpTileStore)
                    uint8_t* ob = stage + 2048;   // result tile
                    const long long row0 = c.grow - lane;
                    if (relu_src != nullptr) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const int r = (lane >> 2) + 8 * k, q = lane & 3;
                            const long long gr = row0 + r;
                            const uint4 u = gr < M ? __ldg(reinterpret_cast<const uint4*>(relu_src + gr * relu_ld + col) + q) : make_uint4(0, 0, 0, 0);
                            *reinterpret_cast<uint4*>(rb + sw64_offset(r, q)) = u;
                        }
                        __syncwarp();
                    }
#pragma unroll
                    for (int j = 0; j < 32; j += 4) {
                        const float4 d4 = lds_f4(sd + ch * 32 + j);
                        x[j] = fmaf(wr, d4.x, x[j]); x[j + 1] = fmaf(wr, d4.y, x[j + 1]);
                        x[j + 2] = fmaf(wr, d4.z, x[j + 2]); x[j + 3] = fmaf(wr, d4.w, x[j + 3]);
                    }
                    if (relu_src != nullptr) {
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const uint4 ru = *reinterpret_cast<const uint4*>(rb + sw64_offset(lane, q));
                            const uint32_t rw[4] = {ru.x, ru.y, ru.z, ru.w};
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const float2 f = unpack_bf16x2(rw[j]);
                                // relu_src is the STORED activation dropout(relu(.)): positive <=> passed the ReLU and was kept, so the
                                // keep-multiplier is the constant scale and no counter hash is drawn (bit-identical to mask * relu')
                                x[q * 8 + 2 * j] = f.x > 0.f ? x[q * 8 + 2 * j] * drop.scale : 0.f;
                                x[q * 8 + 2 * j + 1] = f.y > 0.f ? x[q * 8 + 2 * j + 1] * drop.scale : 0.f;
                            }
                        }
                    } else if (drop.active()) {
                        const uint64_t g0 = (static_cast<uint64_t>(c.grow) * ld + col) >> 2;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            float m[4];
                            drop.mask4_group(g0 + (j >> 2), m);
                            x[j] *= m[0]; x[j + 1] *= m[1]; x[j + 2] *= m[2]; x[j + 3] *= m[3];
                        }
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        *reinterpret_cast<uint4*>(ob + sw64_offset(lane, q)) =
                            make_uint4(pack_bf16x2(x[8 * q], x[8 * q + 1]), pack_bf16x2(x[8 * q + 2], x[8 * q + 3]),
                                       pack_bf16x2(x[8 * q + 4], x[8 * q + 5]), pack_bf16x2(x[8 * q + 6], x[8 * q + 7]));
                    __syncwarp();
                    const int my_orow = v ? static_cast<int>(orow) : -1;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const int r = (lane >> 2) + 8 * k, q = lane & 3;
                        const int orr = __shfl_sync(0xffffffffu, my_orow, r);
                        if (orr >= 0)
                            *(reinterpret_cast<uint4*>(dx + static_cast<long long>(orr) * ld + col) + q) =
                                *reinterpret_cast<const uint4*>(ob + sw64_offset(r, q));
                    }
                    __syncwarp();
                    return;
                }
                if (!v) return;
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const int lc = ch * 32 + g * 8;
                    if (lc >= c.ncols) break;
                    const int col = c.col0 + lc;
                    const int nvalid = min(8, min(c.ncols - lc, N - col));
                    float dd[8];
                    if (lc + 8 <= c.ncols) {
                        const float4 d0 = lds_f4(sd + lc), d1 = lds_f4(sd + lc + 4);
                        dd[0] = d0.x; dd[1] = d0.y; dd[2] = d0.z; dd[3] = d0.w;
                        dd[4] = d1.x; dd[5] = d1.y; dd[6] = d1.z; dd[7] = d1.w;
                    } else {
#pragma unroll
                        for (int j = 0; j < 8; ++j) dd[j] = (j < nvalid) ? lds_f(sd + lc + j) : 0.f;
                    }
                    float y[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) y[j] = (j < nvalid) ? fmaf(wr, dd[j], x[g * 8 + j]) : 0.f;
                    if (relu_src != nullptr) {
                        const uint4 ru = *reinterpret_cast<const uint4*>(relu_src + static_cast<size_t>(c.grow) * relu_ld + col);
                        const uint32_t rw[4] = {ru.x, ru.y, ru.z, ru.w};
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float2 f = unpack_bf16x2(rw[j]);
                            if (!(f.x > 0.f)) y[2 * j] = 0.f;
                            if (!(f.y > 0.f)) y[2 * j + 1] = 0.f;
                        }
                    }
                    if (drop.active()) {
                        float m[8];
                        drop.mask4(c.grow, relu_src != nullptr ? relu_ld : ld, col, m);
                        drop.mask4(c.grow, relu_src != nullptr ? relu_ld : ld, col + 4, m + 4);
#pragma unroll
                        for (int j = 0; j < 8; ++j) y[j] *= m[j];
                    }
                    store_bf16x8(dx + orow * ld + col, y, nvalid);
                }
            });
        if (c.col0 == 0 && c.half == 0 && zero_pad_rows) {  // warp-uniform; the pad rows next to a segment's first / last token
            if ((ld & 7) == 0) {  // the warp zeroes each pad row together (512 contiguous bytes per instruction)
                const int my_orow = static_cast<int>(orow);
                unsigned first = __ballot_sync(0xffffffffu, v && t == 0), last = __ballot_sync(0xffffffffu, v && t == rm.seg_len - 1);
                for (int pass = 0; pass < 2; ++pass) {
                    unsigned m = pass == 0 ? first : last;
                    while (m) {
                        const int src = __ffs(m) - 1;
                        m &= m - 1;
                        const long long prow = __shfl_sync(0xffffffffu, my_orow, src) + (pass == 0 ? -1 : 1);
                        uint4* z = reinterpret_cast<uint4*>(dx + prow * ld);
                        for (int i = lane; i < (ld >> 3); i += 32) z[i] = make_uint4(0, 0, 0, 0);
                    }
                }
            } else if (v) {
                if (t == 0) zero_row_bf16(dx + (orow - 1) * ld, ld);
                if (t == rm.seg_len - 1) zero_row_bf16(dx + (orow + 1) * ld, ld);
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// The same pool backward for an identity row map without a ReLU mask (the self-attention encoders, the additive attention):
//   dX_rc = acc_rc + w_r * dOut[seg(r)][c] [* dropout] -> bf16
// Fragment view, as EpiStore: each warp works on its 16 rows of the tile straight from the wgmma fragment and a whole 32-column
// chunk leaves through a staging box (stmatrix) and TMA; a chunk cut by the slice's end leaves from the fragment with
// predicated stores.  The dOut rows are staged as in EpiDPoolIn.
// scratch: the dOut rows (DOutStage) | the staging boxes (FragStore, 1 KB aligned)
// ------------------------------------------------------------------------------------------------
struct EpiDPoolInFrag {
    static constexpr bool kFragmentView = true;
    using Store = FragStore<6>;
    static constexpr int kScratchBytes = DOutStage::kScratchBytes + Store::kScratchBytes;
    CUtensorMap tm_out;  // dx as a TMA tensor (32 x 16 boxes, SWIZZLE_64B)
    const float* w;      // [rows]
    const float* dout;   // [segments][ldo]
    int ldo;
    int seg_len;
    __nv_bfloat16* dx;   // [rows][ld]
    int ld;
    int N;
    Dropout drop;
    int M;

    __device__ void init(const EpiInit& e, int tile_step) const { DOutStage{dout, ldo, seg_len, M}.init(e, tile_step); }
    __device__ void finish(const EpiInit& e) const { Store::finish(e); }

    __device__ __forceinline__ void frag(const float* acc, const FragCtx& f) const {
        const int lane = threadIdx.x & 31;
        const DOutStage dst{dout, ldo, seg_len, M};
        const float* cur = dst.begin(f.scratch, f.wg, f.it, f.next_tile, f.col0, f.ncols);
        // this lane's rows e = 0, 1: tile row 16 wq + lane / 4 + 8e
        bool v[2];
        float wr[2];
        long long grow[2];
        const float* sd[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int r = 16 * f.wq + (lane >> 2) + 8 * e;
            grow[e] = static_cast<long long>(f.row0) + r;
            v[e] = r < f.rows;
            wr[e] = v[e] ? __ldg(w + grow[e]) : 0.f;
            sd[e] = dst.row(cur, f.row0, f.row0 + r, v[e], f.ncols);
        }
        Store st(f.scratch + DOutStage::kScratchBytes / 4, f, 1);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            if (q < f.nch) {  // a compile-time chunk index keeps the fragment in registers
                const int lc0 = 32 * q;
                float y[16];  // y[4jj + 2e + i]: row e, slice column lc0 + 8jj + 2 (lane % 4) + i
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int lc = lc0 + 8 * jj + 2 * (lane & 3);
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float2 d = lc < f.ncols ? lds_f2(sd[e] + lc) : make_float2(0.f, 0.f);
                        y[4 * jj + 2 * e] = fmaf(wr[e], d.x, acc[16 * q + 4 * jj + 2 * e]);
                        y[4 * jj + 2 * e + 1] = fmaf(wr[e], d.y, acc[16 * q + 4 * jj + 2 * e + 1]);
                    }
                }
                if (drop.active()) drop.apply_frag(y, grow, ld, f.col0 + lc0);
                uint32_t wp[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) wp[k] = pack_bf16x2(y[2 * k], y[2 * k + 1]);
                if (lc0 + 32 <= f.ncols) st.send(&tm_out, wp, f.col0 + lc0);  // warp-uniform; rows >= M are clipped by the tensor map
                else store_frag_bf16(dx, ld, grow, v, f.col0 + lc0, f.ncols - lc0, wp);  // the slice's last chunk
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// Embedding gradient: dEmb[ids[r]][c] += acc_rc [* dropout of the gathered row]; row 0 (padding_idx) skipped
// ------------------------------------------------------------------------------------------------
struct EpiScatter {
    static constexpr int kScratchBytes = 16;
    const long long* ids;  // [rows] token ids (row-mapped through rm for the padded CNN layout)
    float* demb;           // [V][D] fp32
    int V;                 // rows of demb: ids outside [1, V) contribute nothing (the forward gather flags them, the reference
                           // raises IndexError; an unchecked id here would be an out-of-bounds atomic into a neighbouring gradient)
    int D;
    RowMap rm;             // maps the GEMM row to the token index in ids
    Dropout drop;
    int drop_ld;           // pitch used when the forward mask was drawn
    const int* rows;       // null, or compact rows: GEMM row r is token rows[r] (none when negative), its id and dropout row

    __device__ void init(const EpiInit&, int) const {}
    __device__ void finish(const EpiInit&) const {}

    template <class Acc>
    __device__ __forceinline__ void operator()(const Acc& acc, const EpiCtx& c) const {
        long long trow;
        int t;
        bool v;
        int drow = c.grow;  // the row the forward's dropout mask was drawn at
        if (rows != nullptr) {
            drow = c.valid ? rows[c.grow] : -1;
            trow = drow;
            v = drow >= 0;
        } else {
            v = rm.map(c.grow, trow, t) && c.valid;
        }
        long long id = v ? ids[trow] : 0;
        if (id < 0 || id >= V) id = 0;  // out of range: skipped like the padding row
        float* dst = demb + static_cast<size_t>(id) * D;
        epi_chunks(
            acc, c, [](int) {},
            [&](int ch, float* x) {
                if (id == 0) return;
#pragma unroll
                for (int g = 0; g < 8; ++g) {
                    const int lc = ch * 32 + g * 4;
                    if (lc >= c.ncols) break;
                    const int col = c.col0 + lc;
                    float y[4] = {x[g * 4], x[g * 4 + 1], x[g * 4 + 2], x[g * 4 + 3]};
                    if (drop.active()) {
                        float m[4];
                        drop.mask4(drow, drop_ld, col, m);
#pragma unroll
                        for (int j = 0; j < 4; ++j) y[j] *= m[j];
                    }
                    if (col + 4 <= D && lc + 4 <= c.ncols) {
                        red_add_v4_f32(dst + col, y[0], y[1], y[2], y[3]);
                    } else {
                        for (int j = 0; j < 4; ++j)
                            if (col + j < D && lc + j < c.ncols) red_add_f32(dst + col + j, y[j]);
                    }
                }
            });
    }
};

}  // namespace nr
