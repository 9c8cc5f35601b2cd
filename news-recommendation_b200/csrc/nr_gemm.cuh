// Weight-stationary persistent wgmma GEMMs for the news-recommendation hot path (sm_90a).
//
//  gemm_nt : D[M x N] = A[M x K] . B[N x K]^T      (both K-major; "activation x weight^T")
//            * a CTA's weight slice (<=256 output columns, all K, all conv taps) is loaded ONCE by TMA and stays
//              resident in shared memory; 128-row activation tiles stream through a TMA/mbarrier ring; two consumer
//              warpgroups issue wgmma into registers and then run a fused epilogue functor on the accumulator rows.
//            * conv taps: tap s re-loads the A tile shifted by (s - taps/2) rows (zero rows separate
//              the segments in the padded layout), accumulating into the same registers.
//  gemm_tn : D[Ma x Nb] += A[Kr x Ma]^T . B[Kr x Nb]  (both MN-major; weight gradients, Kr = all tokens)
//            split over Kr (and over Nb past 256 columns) across CTAs, fp32 red.global.add epilogue.
//
// Warp roles of gemm_nt (kGemmThreads per CTA): warps 0..kEpiWarps-1 form two warpgroups.  Warpgroup h computes ALL 128
// rows of the tile for its share of the slice's 32-column chunks (the "half" of the epilogue contract) with two m64 wgmmas
// per k-step, so each epilogue thread finds its row and its columns inside its own warpgroup: the row-per-thread view the
// epilogues read is made by passing one 32-column chunk at a time through a small shared-memory transpose buffer.  The
// first warp of the last warpgroup is the TMA producer.
#pragma once
#include "nr_common.cuh"

namespace nr {

constexpr int kEpiWarps = 8;  // gemm_nt epilogue warps: 2 warpgroups (= column parts) x 4 warps (32 rows each)
constexpr int kEpiParts = kEpiWarps / 4;
constexpr int kEpiThreads = kEpiWarps * 32;
// + a producer warpgroup (one warp issues TMA): registers are allocated per warpgroup, and setmaxnreg moves the producer's
// share to the consumers, whose accumulators and epilogue registers need more than the even split of 168
constexpr int kGemmThreads = kEpiThreads + 128;
constexpr int kTnThreads = kGemmThreads;        // gemm_tn: the same two consumer warpgroups + producer
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
constexpr int kTileM = 128;
constexpr int kChunkK = 64;                     // bf16 elements per 128-byte swizzle row
constexpr int kAStageBytes = kTileM * 128;      // 16 KB
constexpr int kMaxStages = 12;
constexpr int kSmemLimit = 232448;              // 227 KB
constexpr int kXposeBytes = kEpiParts * 128 * 16 * 4;  // per warpgroup: 128 rows x 16 fp32 columns (half a chunk)

struct GemmNTParams {
    int M;              // rows of A that exist
    int rows_per_tile;  // rows OWNED by one M tile (<=128); tile t loads rows [t*rpt, t*rpt+128)
    int num_m_tiles;
    int N;              // output columns
    int n_stride;       // columns per weight slice (multiple of 16)
    int n_slices;
    int n_box;          // rows of one resident weight box (multiple of 16, <=256)
    int K;              // reduction length per tap (elements)
    int k_chunks;       // ceil(K/64)
    int taps;           // 1, or 3 for the window-3 title CNN
    int b_tap_rows;     // row offset between taps inside the weight operand
    int stages;
    int b_stream;       // 1: the weight slice does not fit beside the ring; its (tap, k-chunk) box travels with every A stage
    int stage_bytes;    // kAStageBytes (+ one weight box when b_stream)
    float* dbg_acc;     // debug backend only: fp32 accumulators [num_m_tiles*128][dbg_ld]
    int dbg_ld;
    int dbg_flags;      // tuning only (NEWSREC_GEMM_DBG): bit 1 = the producer skips the A loads (MMA on stale data)
    long long* timing;  // tuning only (nr_debug_set_gemm_timing): per CTA 16 cycle counters, see the kernel
};

// What an epilogue functor sees for one (tile,row).
struct EpiCtx {
    int tile;
    int r;        // row inside the tile (0..127)
    int grow;     // global A row
    bool valid;   // r < rows_per_tile && grow < M
    int col0;     // first output column of this CTA's slice
    int ncols;    // valid output columns in the slice
    int tid;      // 0..255 within the epilogue group
    int half;     // 0 .. kEpiParts-1: column part (= warpgroup)
    int ch0, ch1; // this thread's range of 32-column chunks
    float* scratch;  // Epi::kScratchBytes of shared memory private to the epilogue group
    int it;          // how many tiles this CTA has finished before this one (double-buffer parity of the epilogue staging)
    int next_tile;   // the tile this CTA processes next, or -1
};
// What init()/finish() see.
struct EpiInit {
    int col0, ncols, tid;
    float* scratch;
    int first_tile;  // first tile of this CTA (>= num_tiles: the CTA has no work)
    int num_tiles;
};

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory"); }
// the two column halves run different chunk counts: barriers inside a chunk loop are per half

__device__ __forceinline__ void epi_chunk_range(int ncols, int part, int& ch0, int& ch1) {
    const int nch = (ncols + 31) >> 5, base = nch / kEpiParts, rem = nch - base * kEpiParts;
    ch0 = part * base + min(part, rem);
    ch1 = ch0 + base + (part < rem ? 1 : 0);
}

// Accumulators of one warpgroup: acc[b] is the m64 wgmma fragment of rows [64b, 64b + 64) for the warpgroup's chunks
// [ch0, ch1) (at most 4).  load32(ch) hands every thread the 32 columns of chunk ch of its own row (row = thread of the
// warpgroup), through the warpgroup's transpose buffer, 16 columns at a time; every thread of the warpgroup calls it with the
// same chunk sequence (the chunk range is per warpgroup).  Buffer layout: row r, column c at r*16 + ((c/4) ^ ((r/2)&3))*4 + c%4
// (conflict-free row reads).
struct RegAcc {
    float (*acc)[64];
    float* xpose;   // this warpgroup's 8 KB
    int ch0;
    int bar_id;     // named barrier of the warpgroup
    __device__ __forceinline__ void sync() const { asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory"); }
    template <int Q>
    __device__ __forceinline__ void put_half(int hf) const {  // columns [32Q + 16hf, +16) of the fragment into the buffer
        const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                const int j = 4 * Q + 2 * hf + jj;  // 8-column group of the fragment
                const int c = 8 * jj + 2 * (lane & 3);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int r = 64 * b + 16 * wq + (lane >> 2) + 8 * e;
                    *reinterpret_cast<float2*>(xpose + r * 16 + (((c >> 2) ^ ((r >> 1) & 3)) << 2) + (c & 3)) =
                        make_float2(acc[b][4 * j + 2 * e], acc[b][4 * j + 2 * e + 1]);
                }
            }
    }
    __device__ __forceinline__ void load32(int chunk, float* v) const {
        const int q = chunk - ch0, r = threadIdx.x & 127;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            sync();  // every thread has read the previous half out of the buffer
            switch (q) {
                case 0: put_half<0>(hf); break;
                case 1: put_half<1>(hf); break;
                case 2: put_half<2>(hf); break;
                default: put_half<3>(hf); break;
            }
            sync();
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const float4 f = lds_f4(xpose + r * 16 + ((g ^ ((r >> 1) & 3)) << 2));
                v[16 * hf + 4 * g] = f.x; v[16 * hf + 4 * g + 1] = f.y; v[16 * hf + 4 * g + 2] = f.z; v[16 * hf + 4 * g + 3] = f.w;
            }
        }
    }
    __device__ __forceinline__ void release() const {}
};
struct GlobalAcc {  // debug backend: accumulators computed by a plain SIMT kernel
    const float* row;
    __device__ __forceinline__ void load32(int chunk, float* v) const {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = row[chunk * 32 + j];
    }
    __device__ __forceinline__ void release() const {}
};

// The chunk loop every epilogue shares.  pre(ch) runs before the load of chunk ch (shared-memory operand loads go there).
// Calls acc.release() exactly once, after the last chunk has landed in registers.
template <class Acc, class Pre, class Body>
__device__ __forceinline__ void epi_chunks(const Acc& acc, const EpiCtx& c, Pre&& pre, Body&& body) {
    for (int ch = c.ch0; ch < c.ch1; ++ch) {
        float x[32];
        pre(ch);
        acc.load32(ch, x);
        if (ch + 1 == c.ch1) acc.release();
        body(ch, x);
    }
    if (c.ch0 >= c.ch1) acc.release();
}

// bf16 output tiles leave through TMA instead of 32 scattered rows per store instruction: a warp packs its 32 rows x 32
// columns into a private staging buffer (SWIZZLE_64B layout: 16-byte chunk q of row r at r*64 + ((q ^ (r>>1)) & 3)*16,
// conflict-free for row-per-lane 16-byte writes) and one lane issues cp.async.bulk.tensor.  Two buffers per warp.
// Row-per-thread stores of 32 rows sit in the LSU queue and stall the warps on their source registers.
constexpr int kTileStoreBufs = 2;                                  // staging tiles per warp (2 KB each)
constexpr int kTileStoreBytes = kEpiWarps * kTileStoreBufs * 2048 + 1024;  // + alignment slack
struct WarpTileStore {
    uint8_t* buf;  // this warp's kTileStoreBufs x 2 KB (1024-byte aligned)
    int nput;
    __device__ __forceinline__ void attach(void* region, int warp_in_group) {
        buf = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(region) + 1023) & ~uintptr_t(1023)) + warp_in_group * (kTileStoreBufs * 2048);
    }
    __device__ __forceinline__ void begin_tile(int lane) {
        nput = 0;
        if (lane == 0) bulk_wait_read<0>();
        __syncwarp();
    }
    // w: this lane's row, 32 columns as 16 packed bf16 pairs; (col, row0) = global coordinates of the warp's tile
    __device__ __forceinline__ void put(const CUtensorMap* tm, const uint32_t* w, int col, int row0, int lane) {
        uint8_t* b = buf + (nput % kTileStoreBufs) * 2048;
        if (nput >= kTileStoreBufs) {
            if (lane == 0) bulk_wait_read<kTileStoreBufs - 1>();  // the store issued from this buffer has been read out
            __syncwarp();
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
            *reinterpret_cast<uint4*>(b + lane * 64 + ((q ^ (lane >> 1)) & 3) * 16) =
                make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
            tma_store_2d(tm, b, col, row0);
            bulk_commit();
        }
        ++nput;
    }
    // Row-mapped destinations (no tensor map fits them): the same staging tile leaves as coalesced 16-byte stores, 8 rows x 64
    // contiguous bytes per instruction.  my_orow = destination row of this lane's accumulator row, -1 for "drop the row".
    __device__ __forceinline__ void put_rows(__nv_bfloat16* base, int ld, const uint32_t* w, int col, int my_orow, int lane) {
        uint8_t* b = buf;
#pragma unroll
        for (int q = 0; q < 4; ++q)
            *reinterpret_cast<uint4*>(b + lane * 64 + ((q ^ (lane >> 1)) & 3) * 16) =
                make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int r = (lane >> 2) + 8 * k, q = lane & 3;
            const int orr = __shfl_sync(0xffffffffu, my_orow, r);
            if (orr >= 0)
                *(reinterpret_cast<uint4*>(base + static_cast<long long>(orr) * ld + col) + q) =
                    *reinterpret_cast<const uint4*>(b + r * 64 + ((q ^ (r >> 1)) & 3) * 16);
        }
        __syncwarp();
    }
    static __device__ __forceinline__ void drain(int lane) {  // before the CTA exits
        if (lane == 0) bulk_wait_all();
    }
};

// ---------------------------------------------------------------------------------------------
// gemm_nt kernel: one CTA per (tile sequence, weight slice)
// ---------------------------------------------------------------------------------------------
// mbarrier protocol:
//   bfull     count 1 + tx of the resident weight slice    -> the consumers may start (not used when b_stream)
//   full[s]   count 1 + tx of one A box (+ its weight box when b_stream; the producer's expect_tx)
//   empty[s]  count kEpiWarps: every consumer warp arrives once its wgmmas on stage s have completed
// Warpgroup h multiplies the 128-row A tile by the weight rows of its chunks [ch0, ch1): two m64 x (32 * nch) wgmmas per
// k-step, nch <= 4 (a slice is <= 256 columns, split into two parts).
// The MMAs of one tile for a warpgroup with NCH chunks (a compile-time N keeps the wgmmas asynchronous): one wgmma group
// per ring stage, one group left in flight while the next stage is awaited; a stage is released once its group completed.
template <int NCH>
__device__ __forceinline__ void gemm_nt_mma_tile(float (*acc)[64], const GemmNTParams& p, uint64_t* full, uint64_t* empty,
                                                 int& st, uint32_t& ph, uint32_t a_s, uint32_t b_s, uint32_t b_off, int b_region,
                                                 int lane) {
    int prev = -1;
    for (int s = 0; s < p.taps; ++s)
        for (int kc = 0; kc < p.k_chunks; ++kc) {
            mbar_wait(&full[st], ph, 104);
            if constexpr (NCH > 0) {
                const uint32_t a_st = a_s + st * p.stage_bytes;
                const uint32_t b_box = p.b_stream ? a_st + kAStageBytes + b_off : b_s + (s * p.k_chunks + kc) * b_region;
                const uint64_t db = make_sw128_desc(b_box, 16, 1024);
                const int first = (s | kc) == 0;
#pragma unroll
                for (int b = 0; b < 2; ++b)
#pragma unroll
                    for (int i = 0; i < 16 * NCH; ++i) wgmma_reg_fence(acc[b][i]);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)  // +32 bytes per k-step = +2 in the descriptor's >>4 address field
#pragma unroll
                    for (int b = 0; b < 2; ++b)
                        Wgmma<32 * NCH, 0, 0>::mma(acc[b], make_sw128_desc(a_st + b * 8192, 16, 1024) + 2 * k, db + 2 * k,
                                                   (first && k == 0) ? 0 : 1);
                wgmma_commit();
                wgmma_wait<1>();  // the group of the previous stage has completed
            }
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);  // this warp's reads of stage prev are complete
            }
            prev = st;
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
    if constexpr (NCH > 0) {
        wgmma_wait<0>();
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int i = 0; i < 16 * NCH; ++i) wgmma_reg_fence(acc[b][i]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);
}

template <class Epi>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_nt_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmNTParams p,
               const __grid_constant__ Epi epi) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    const int b_region = p.n_box * 128;  // bytes of one (tap, k-chunk) box of the weight slice
    uint8_t* sB = smem;
    uint8_t* sA = sB + (p.b_stream ? 0 : p.taps * p.k_chunks * b_region);
    float* xpose = reinterpret_cast<float*>(sA + p.stages * p.stage_bytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(xpose) + kXposeBytes);
    uint64_t* full = bars;
    uint64_t* empty = bars + kMaxStages;
    uint64_t* bfull = bars + 2 * kMaxStages;
    float* scratch = reinterpret_cast<float*>(bars + 2 * kMaxStages + 8);

    const int slice = blockIdx.x % p.n_slices;
    const int tile0 = blockIdx.x / p.n_slices;
    const int tile_step = gridDim.x / p.n_slices;
    const int col0 = slice * p.n_stride;
    const int ncols = min(p.n_stride, p.N - col0);
    const int tap_shift = p.taps / 2;
    // tuning counters: [0] producer waits for a free A stage, [1] MMA loops incl. waits for A data, [4] epilogue body, [5] kernel,
    // [6] tiles
    long long* tmr = p.timing != nullptr ? p.timing + blockIdx.x * 16 : nullptr;
    const long long t_begin = tmr != nullptr ? clock64() : 0;
    long long tw_a = 0, tw_b = 0;
    auto timed_wait = [&](uint64_t* bar, uint32_t parity, int code, long long& acc_t) {
        if (tmr != nullptr) {
            const long long t = clock64();
            mbar_wait(bar, parity, code);
            acc_t += clock64() - t;
        } else {
            mbar_wait(bar, parity, code);
        }
    };

    if (warp == kEpiWarps && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], kEpiWarps);
        }
        mbar_init(bfull, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= kEpiWarps) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
        if (warp != kEpiWarps) return;
        // ===================== TMA producer (uniform loops, one elected lane issues) =====================
        if (!p.b_stream && elect_one()) {
            mbar_arrive_expect_tx(bfull, static_cast<uint32_t>(p.taps * p.k_chunks * b_region));
            for (int s = 0; s < p.taps; ++s)
                for (int kc = 0; kc < p.k_chunks; ++kc)
                    tma_load_2d(sB + (s * p.k_chunks + kc) * b_region, &tmB, bfull, kc * kChunkK, s * p.b_tap_rows + col0);
        }
        __syncwarp();
        int st = 0;
        uint32_t ph = 0;
        for (int tile = tile0; tile < p.num_m_tiles; tile += tile_step) {
            const int row0 = tile * p.rows_per_tile;
            for (int s = 0; s < p.taps; ++s)
                for (int kc = 0; kc < p.k_chunks; ++kc) {
                    timed_wait(&empty[st], ph ^ 1, 101, tw_a);
                    if (elect_one()) {
#ifdef NEWSREC_TRIAGE
                        if (p.dbg_flags & 2) {
                            mbar_arrive(&full[st]);
                        } else
#endif
                        {
                            mbar_arrive_expect_tx(&full[st], p.stage_bytes);
                            tma_load_2d(sA + st * p.stage_bytes, &tmA, &full[st], kc * kChunkK, row0 + s - tap_shift);  // rows past M / before 0: zero filled
                            if (p.b_stream)
                                tma_load_2d(sA + st * p.stage_bytes + kAStageBytes, &tmB, &full[st], kc * kChunkK, s * p.b_tap_rows + col0);
                        }
                    }
                    __syncwarp();
                    if (++st == p.stages) { st = 0; ph ^= 1; }
                }
        }
        if (tmr != nullptr && lane == 0) tmr[0] = tw_a;
    } else {
        // ===================== consumer warpgroups: wgmma, then the epilogue on the same registers =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
        const int half = warp >> 2;
        const int quarter = warp & 3;
        int ch0, ch1;
        epi_chunk_range(ncols, half, ch0, ch1);
        const int nch = ch1 - ch0;
        const EpiInit ei{col0, ncols, static_cast<int>(threadIdx.x), scratch, tile0, p.num_m_tiles};
        epi.init(ei, tile_step);
        const uint32_t a_s = smem_u32(sA), b_s = smem_u32(sB) + ch0 * 32 * 128;
        const uint32_t b_off = ch0 * 32 * 128;
        float acc[2][64];
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[b][i] = 0.f;
        const RegAcc racc{acc, xpose + half * (kXposeBytes / 4 / kEpiParts), ch0, 2 + half};
        if (!p.b_stream) mbar_wait(bfull, 0, 102);
        int st = 0;
        uint32_t ph = 0;
        int it = 0;
        for (int tile = tile0; tile < p.num_m_tiles; tile += tile_step, ++it) {
            const long long t_mma = tmr != nullptr ? clock64() : 0;
            switch (nch) {
                case 0: gemm_nt_mma_tile<0>(acc, p, full, empty, st, ph, a_s, b_s, b_off, b_region, lane); break;
                case 1: gemm_nt_mma_tile<1>(acc, p, full, empty, st, ph, a_s, b_s, b_off, b_region, lane); break;
                case 2: gemm_nt_mma_tile<2>(acc, p, full, empty, st, ph, a_s, b_s, b_off, b_region, lane); break;
                case 3: gemm_nt_mma_tile<3>(acc, p, full, empty, st, ph, a_s, b_s, b_off, b_region, lane); break;
                default: gemm_nt_mma_tile<4>(acc, p, full, empty, st, ph, a_s, b_s, b_off, b_region, lane); break;
            }
            if (tmr != nullptr) tw_b += clock64() - t_mma;
            const long long t_epi = tmr != nullptr ? clock64() : 0;
            EpiCtx c;
            c.tile = tile;
            c.r = quarter * 32 + lane;
            c.grow = tile * p.rows_per_tile + c.r;
            c.valid = (c.r < p.rows_per_tile) && (c.grow < p.M);
            c.col0 = col0;
            c.ncols = ncols;
            c.tid = threadIdx.x;
            c.half = half;
            c.ch0 = ch0;
            c.ch1 = ch1;
            c.scratch = scratch;
            c.it = it;
            c.next_tile = tile + tile_step < p.num_m_tiles ? tile + tile_step : -1;
            epi(racc, c);
            if (tmr != nullptr) tw_a += clock64() - t_epi;
        }
        epi.finish(ei);
        if (tmr != nullptr && threadIdx.x == 0) { tmr[1] = tw_b; tmr[4] = tw_a; tmr[5] = clock64() - t_begin; tmr[6] = it; }
    }
}

// Debug backend (TRIAGE builds only -- `make TRIAGE=1`, -DNEWSREC_TRIAGE; the release library has no second backend and
// consults no environment switch on the launch path): plain SIMT accumulate + the SAME epilogue functors.
#ifdef NEWSREC_TRIAGE
__global__ void gemm_nt_simt_acc_kernel(const __nv_bfloat16* A, int lda, const __nv_bfloat16* B, int ldb,
                                        GemmNTParams p);
template <class Epi>
__global__ void __launch_bounds__(kEpiThreads, 1) gemm_nt_simt_epi_kernel(const GemmNTParams p, const __grid_constant__ Epi epi) {
    extern __shared__ __align__(1024) float scratch[];  // Epi::kScratchBytes
    const int slice = blockIdx.x % p.n_slices;
    const int tile0 = blockIdx.x / p.n_slices;
    const int tile_step = gridDim.x / p.n_slices;
    const int col0 = slice * p.n_stride;
    const int ncols = min(p.n_stride, p.N - col0);
    for (int i = threadIdx.x; i < Epi::kScratchBytes / 4; i += kEpiThreads) scratch[i] = 0.f;
    __syncthreads();
    const EpiInit ei{col0, ncols, static_cast<int>(threadIdx.x), scratch, tile0, p.num_m_tiles};
    epi.init(ei, tile_step);
    int it = 0;
    for (int tile = tile0; tile < p.num_m_tiles; tile += tile_step, ++it) {
        EpiCtx c;
        c.tile = tile;
        c.r = threadIdx.x & 127;
        c.grow = tile * p.rows_per_tile + c.r;
        c.valid = (c.r < p.rows_per_tile) && (c.grow < p.M);
        c.col0 = col0;
        c.ncols = ncols;
        c.tid = threadIdx.x;
        c.half = threadIdx.x >> 7;
        epi_chunk_range(ncols, c.half, c.ch0, c.ch1);
        c.scratch = scratch;
        c.it = it;
        c.next_tile = tile + tile_step < p.num_m_tiles ? tile + tile_step : -1;
        GlobalAcc acc{p.dbg_acc + (static_cast<size_t>(tile) * 128 + c.r) * p.dbg_ld + col0};
        epi(acc, c);
    }
    epi.finish(ei);
}
#endif  // NEWSREC_TRIAGE

// ---------------------------------------------------------------------------------------------
// gemm_tn kernel
// ---------------------------------------------------------------------------------------------
struct GemmTNParams {
    int Kr;          // reduction rows (tokens)
    int Ma;          // output rows  = columns of A
    int Nb;          // output cols  = columns of B used (<=512)
    int b_col0;      // first B column
    int b_row_shift; // B row = A row + shift (conv taps)
    int m_tiles;
    int n_tiles;     // CTAs along Nb (<= 256 columns each)
    int k_slices;
    int chunks_per_slice;  // 64-row chunks per CTA
    int n_boxes;     // ceil(Nb/64)
    int stages;
    float* D;        // fp32 [Ma][ldd], accumulated with red.global.add
    int ldd;
};


// ---------------------------------------------------------------------------------------------
// host-side launch helpers (gemm.cu)
// ---------------------------------------------------------------------------------------------
struct GemmNTPlan {
    GemmNTParams p;
    CUtensorMap tmA, tmB;
    int grid;
    size_t smem;
};
// Fills slices/boxes/stages and encodes the tensor maps.  A: [M rows][K] pitch lda; B: [taps*b_tap_rows][K] pitch ldb.
// scratch_bytes = Epi::kScratchBytes; max_n_stride (0 = none) caps the slice width for epilogues whose staging
// grows with it.
int plan_gemm_nt(GemmNTPlan* plan, const void* A, int M, int lda, const void* B, int N, int ldb, int K, int taps,
                 int b_tap_rows, int rows_per_tile, int num_sms, int max_slices, int scratch_bytes, int max_n_stride);
bool debug_simt_gemm();

template <class Epi>
int launch_gemm_nt(const GemmNTPlan& plan, const Epi& epi, const void* A, int lda, const void* B, int ldb,
                   cudaStream_t stream) {
    if (plan.p.num_m_tiles <= 0) return 0;
#ifdef NEWSREC_TRIAGE
    if (debug_simt_gemm()) {
        GemmNTParams p = plan.p;
        const size_t ld = static_cast<size_t>(round_up(p.N, 32) + 32);
        float* acc = nullptr;
        NR_CHECK_CUDA(cudaMallocAsync(&acc, sizeof(float) * ld * p.num_m_tiles * 128, stream));
        p.dbg_acc = acc;
        p.dbg_ld = static_cast<int>(ld);
        dim3 g(ceil_div(static_cast<int>(ld), 128), p.num_m_tiles);
        gemm_nt_simt_acc_kernel<<<g, 128, 0, stream>>>(static_cast<const __nv_bfloat16*>(A), lda,
                                                       static_cast<const __nv_bfloat16*>(B), ldb, p);
        static bool dbg_attr_set = false;  // per Epi instantiation
        if (!dbg_attr_set) {
            NR_CHECK_CUDA(cudaFuncSetAttribute(gemm_nt_simt_epi_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               Epi::kScratchBytes));
            dbg_attr_set = true;
        }
        gemm_nt_simt_epi_kernel<Epi><<<plan.grid, kEpiThreads, Epi::kScratchBytes, stream>>>(p, epi);
        NR_CHECK_CUDA(cudaGetLastError());
        NR_CHECK_CUDA(cudaFreeAsync(acc, stream));
        return 0;
    }
#endif
    static bool attr_set = false;  // per Epi instantiation
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(gemm_nt_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
        attr_set = true;
    }
    gemm_nt_kernel<Epi><<<plan.grid, kGemmThreads, plan.smem, stream>>>(plan.tmA, plan.tmB, plan.p, epi);
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// D[Ma x Nb] (+)= A[:, 0:Ma]^T . B[shifted rows, b_col0 : b_col0+Nb]
int launch_gemm_tn(const void* A, int Kr, int Ma, int lda, const void* B, int b_rows, int b_cols, int ldb, int b_col0,
                   int Nb, int b_row_shift, float* D, int ldd, int num_sms, cudaStream_t stream);

int num_sms();
extern int g_launches;  // kernels launched by this library (bench.py reports it)

}  // namespace nr
