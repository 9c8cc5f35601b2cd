// Weight-stationary persistent wgmma GEMMs for the news-recommendation hot path (sm_90a).
//
//  gemm_nt : D[M x N] = A[M x K] . B[N x K]^T      (both K-major; "activation x weight^T")
//            * a CTA's weight slice (<=256 output columns, all K, all conv taps) is loaded ONCE by TMA and stays
//              resident in shared memory; 64-row activation tiles stream through a TMA/mbarrier ring; two consumer
//              warpgroups take the CTA's tiles in turn and run a fused epilogue functor on the accumulator rows.
//            * conv taps: tap s re-loads the A tile shifted by (s - tap_origin) rows (tap_origin = taps/2 for the centred
//              window, whose padded layout separates the segments by zero rows), accumulating into the same registers.
//  gemm_tn : D[Ma x Nb] += A[Kr x Ma]^T . B[Kr x Nb]  (both MN-major; weight gradients, Kr = all tokens)
//            split over Kr (and over Nb past 256 columns) across CTAs, fp32 red.global.add epilogue.
//
// Warp roles of gemm_nt (kGemmThreads per CTA): warps 0..kEpiWarps-1 form two consumer warpgroups, the first warp of the
// last warpgroup is the TMA producer.  Ping-pong schedule: warpgroup w owns the CTA's tiles w, w + 2, w + 4, ... and computes
// a whole tile (64 rows x the whole slice) with one m64nN wgmma per k-step, N = 32 * (chunks of the slice).  The two
// warpgroups issue their MMAs in strict alternation (a pair of named barriers passes the tensor pipe from one to the other),
// so one warpgroup's epilogue runs while the other's wgmmas execute.  An epilogue takes one of two views of the accumulators:
//   * fragment view (Epi::kFragmentView): each warp reads its 16 rows of the m64 fragment in registers, with no shared memory
//     and no barrier across warps -- for epilogues whose output elements are independent (EpiStore);
//   * row view: row-per-thread, the fragment passes through a small shared-memory transpose buffer one 32-column chunk per
//     column half at a time -- for epilogues that reduce along a row or a column.
#pragma once
#include "nr_common.cuh"

namespace nr {

constexpr int kEpiWarps = 8;    // gemm_nt consumer / epilogue warps: 2 warpgroups, each owning whole tiles
constexpr int kEpiThreads = kEpiWarps * 32;
constexpr int kWgThreads = 128;
constexpr int kEpiHalves = 2;   // column halves of a warpgroup's epilogue: warps 0-1 and 2-3 of the warpgroup
// + a producer warpgroup (one warp issues TMA): registers are allocated per warpgroup, and setmaxnreg moves the producer's
// share to the consumers, whose accumulators and epilogue registers need more than the even split of 168
constexpr int kGemmThreads = kEpiThreads + 128;
constexpr int kTnThreads = kGemmThreads;        // gemm_tn: the same two consumer warpgroups + producer
constexpr int kProducerRegs = 40, kConsumerRegs = 232;  // gemm_tn
// gemm_nt: a consumer holds a whole m64n256 fragment (128 registers) next to its epilogue's; the TMA producer needs few
constexpr int kNtProducerRegs = 24, kNtConsumerRegs = 240;
constexpr int kTileM = 64;                      // gemm_nt rows per tile: one m64 wgmma
constexpr int kChunkK = 64;                     // bf16 elements per 128-byte swizzle row
constexpr int kAStageBytes = kTileM * 128;      // 8 KB
constexpr int kMaxStages = 12;
constexpr int kSmemLimit = 232448;              // 227 KB
constexpr int kXposeBytes = 2 * kEpiHalves * kTileM * 16 * 4;  // row view: per warpgroup and column half 64 rows x 16 fp32 columns
// named barriers of gemm_nt (0 is __syncthreads): all consumer threads, each warpgroup's own, each warpgroup's MMA turn
constexpr int kBarConsumers = 1, kBarWg = 2, kBarTurn = 4;

struct GemmNTParams {
    int M;              // rows of A that exist
    int rows_per_tile;  // rows OWNED by one M tile (<=64); tile t loads rows [t*rpt, t*rpt+64)
    int num_m_tiles;
    int N;              // output columns
    int n_stride;       // columns per weight slice (multiple of 16)
    int n_slices;
    int n_box;          // rows of one resident weight box (multiple of 32, <=256)
    int K;              // reduction length per tap (elements)
    int k_chunks;       // ceil(K/64)
    int taps;           // 1 .. 4 conv taps (3 for the window-3 title CNN)
    int tap_origin;     // tap s reads A rows shifted by s - tap_origin (plan_gemm_nt: taps / 2)
    int b_tap_rows;     // row offset between taps inside the weight operand
    int stages;
    int b_stream;       // 1: the weight slice does not fit beside the ring; its (tap, k-chunk) box travels with every A stage
    int stage_bytes;    // kAStageBytes (+ one weight box when b_stream)
    // null: every tile 0 .. num_m_tiles-1.  Otherwise the tiles to process, written on the device before the launch:
    // tile_list[0] = their count, tile_list[1 ..] = the tiles in ascending order.  The CTAs stride over list positions the way
    // they stride over tiles without a list; a CTA whose first position is past the count leaves at once.
    const int* tile_list;
    float* dbg_acc;     // debug backend only: fp32 accumulators [num_m_tiles*kTileM][dbg_ld]
    int dbg_ld;
    int dbg_flags;      // tuning only (NEWSREC_GEMM_DBG): bit 1 = the producer skips the A loads (MMA on stale data)
    long long* timing;  // tuning only (nr_debug_set_gemm_timing): per CTA 16 cycle counters, see the kernel
};

// What an epilogue functor sees for one (tile,row).
struct EpiCtx {
    int tile;
    int r;        // row inside the tile (0..63)
    int grow;     // global A row
    bool valid;   // r < rows_per_tile && grow < M
    int col0;     // first output column of this CTA's slice
    int ncols;    // valid output columns in the slice
    int tid;      // 0..255 over both consumer warpgroups (warp tid/32 owns 32 rows of its warpgroup's tile)
    int wg;       // consumer warpgroup (0, 1) that owns this tile
    int wtid;     // 0..127 within the warpgroup
    int half;     // 0 .. kEpiHalves-1: column half inside the warpgroup
    int ch0, ch1; // this thread's range of 32-column chunks
    int rounds;   // collective chunk loads per tile (the larger half's chunk count)
    float* scratch;  // Epi::kScratchBytes of shared memory private to the epilogue (both warpgroups)
    int it;          // how many tiles this warpgroup has finished before this one (double-buffer parity of the staging)
    int next_tile;   // the tile this warpgroup processes next, or -1
};
// What a fragment-view epilogue sees for one tile: frag(acc, f) is called by every thread of the warpgroup that owns the
// tile, acc is its m64nN fragment (acc[4j + 2e + i] = tile row 16 * wq + lane / 4 + 8e, slice column 8j + 2 * (lane % 4) + i,
// j < 4 * nch).
struct FragCtx {
    int row0;     // global A row of the tile's row 0
    int rows;     // rows of the tile that exist (r < rows: rows_per_tile, fewer at the end of A)
    int wq;       // warp in the warpgroup
    int nch;      // 32-column chunks of the slice
    int col0;     // first output column of this CTA's slice
    int ncols;    // valid output columns in the slice
    float* scratch;  // Epi::kScratchBytes of shared memory private to the epilogue (both warpgroups)
    int wg;          // consumer warpgroup (0, 1) that owns this tile
    int it;          // how many tiles this warpgroup has finished before this one (double-buffer parity of the staging)
    int next_tile;   // the tile this warpgroup processes next, or -1
};
template <class Epi>
concept FragmentEpilogue = Epi::kFragmentView;
// shared memory an epilogue needs beside the pipeline: its scratch, plus the transpose buffers of the row view
template <class Epi>
constexpr int kEpiSmemBytes = Epi::kScratchBytes + (FragmentEpilogue<Epi> ? 0 : kXposeBytes);

// What init()/finish() see (all kEpiThreads consumer threads call them).
struct EpiInit {
    int col0, ncols, tid;
    float* scratch;
    int first_tile;  // first tile of this CTA (warpgroup w starts at first_tile + w * tile_step); a list position with a tile list
    int num_tiles;
};

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// init()/finish(): every consumer thread of the CTA
__device__ __forceinline__ void consumers_bar_sync() { named_bar_sync(kBarConsumers, kEpiThreads); }
// per tile: the threads of the warpgroup that owns it (the two column halves run different chunk counts: barriers inside a
// chunk loop are per half)
__device__ __forceinline__ void epi_bar_sync(int wg) { named_bar_sync(kBarWg + wg, kWgThreads); }

__device__ __forceinline__ void epi_chunk_range(int ncols, int part, int& ch0, int& ch1) {
    const int nch = (ncols + 31) >> 5, base = nch / kEpiHalves, rem = nch - base * kEpiHalves;
    ch0 = part * base + min(part, rem);
    ch1 = ch0 + base + (part < rem ? 1 : 0);
}

// Accumulators of one warpgroup: the m64nN wgmma fragment of its tile (acc[4j + 2e + i] = row 16 * (warp % 4) + lane / 4 + 8e,
// column 8j + 2 * (lane % 4) + i).  Thread t of the warpgroup reads row 32 * ((t / 32) % 2) + t % 32 of column half t / 64:
// half 0 owns chunks [0, second), half 1 chunks [second, nch).  load32(i) is collective over the warpgroup: round i hands
// every thread the 32 columns of its half's i-th chunk, through the warpgroup's transpose buffers (one per half, 64 rows x
// 16 columns), 16 columns at a time; when nch is odd, half 1 has no chunk in the last round and only reads.  Buffer layout:
// row r, column c at r*16 + ((c/4) ^ ((r/2)&3))*4 + c%4 (conflict-free row reads).
struct RegAcc {
    float* acc;
    float* xpose;   // this warpgroup's 8 KB
    int second;     // first chunk of column half 1 (= the number of rounds)
    int nch;
    int bar_id;     // named barrier of the warpgroup
    __device__ __forceinline__ void sync() const { named_bar_sync(bar_id, kWgThreads); }
    template <int Q>
    __device__ __forceinline__ void put_half(int hf, float* buf) const {  // columns [32Q + 16hf, +16) of the fragment
        const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int j = 4 * Q + 2 * hf + jj;  // 8-column group of the fragment
            const int c = 8 * jj + 2 * (lane & 3);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int r = 16 * wq + (lane >> 2) + 8 * e;
                *reinterpret_cast<float2*>(buf + r * 16 + (((c >> 2) ^ ((r >> 1) & 3)) << 2) + (c & 3)) =
                    make_float2(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]);
            }
        }
    }
    __device__ __forceinline__ void put_chunk(int q, int hf, float* buf) const {
        switch (q) {
            case 0: put_half<0>(hf, buf); break;
            case 1: put_half<1>(hf, buf); break;
            case 2: put_half<2>(hf, buf); break;
            case 3: put_half<3>(hf, buf); break;
            case 4: put_half<4>(hf, buf); break;
            case 5: put_half<5>(hf, buf); break;
            case 6: put_half<6>(hf, buf); break;
            default: put_half<7>(hf, buf); break;
        }
    }
    __device__ __forceinline__ void load32(int i, float* v) const {
        const int t = threadIdx.x & 127, r = 32 * ((t >> 5) & 1) + (t & 31);
        const float* mine = xpose + (t >> 6) * (kTileM * 16);
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            sync();  // every thread has read the previous half out of the buffers
            put_chunk(i, hf, xpose);
            if (second + i < nch) put_chunk(second + i, hf, xpose + kTileM * 16);
            sync();
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const float4 f = lds_f4(mine + r * 16 + ((g ^ ((r >> 1) & 3)) << 2));
                v[16 * hf + 4 * g] = f.x; v[16 * hf + 4 * g + 1] = f.y; v[16 * hf + 4 * g + 2] = f.z; v[16 * hf + 4 * g + 3] = f.w;
            }
        }
    }
    __device__ __forceinline__ void release() const {}
};
struct GlobalAcc {  // debug backend: accumulators computed by a plain SIMT kernel
    const float* row;
    int ch0, ch1;
    __device__ __forceinline__ void load32(int i, float* v) const {
        const int chunk = ch0 + i;
        if (chunk >= ch1) return;
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = row[chunk * 32 + j];
    }
    __device__ __forceinline__ void release() const {}
};

// The chunk loop every epilogue shares: c.rounds collective loads, the thread's chunk of round i is ch0 + i (when it has one).
// pre(ch) runs before the load of chunk ch (shared-memory operand loads go there).  Calls acc.release() exactly once, after
// the last chunk has landed in registers.
template <class Acc, class Pre, class Body>
__device__ __forceinline__ void epi_chunks(const Acc& acc, const EpiCtx& c, Pre&& pre, Body&& body) {
    for (int i = 0; i < c.rounds; ++i) {
        const int ch = c.ch0 + i;
        const bool mine = ch < c.ch1;  // warp-uniform
        float x[32];
        if (mine) pre(ch);
        acc.load32(i, x);
        if (mine) body(ch, x);
    }
    acc.release();
}

// Tiles a gemm_nt launch processes, and the tile at list position i (see GemmNTParams::tile_list)
__device__ __forceinline__ int gemm_nt_tile_count(const GemmNTParams& p) { return p.tile_list != nullptr ? p.tile_list[0] : p.num_m_tiles; }
__device__ __forceinline__ int gemm_nt_tile_at(const GemmNTParams& p, int i) { return p.tile_list != nullptr ? p.tile_list[1 + i] : i; }

// What the calling consumer thread's epilogue sees of the tile at list position i, the it-th tile of its warpgroup (both
// gemm_nt back-ends; n_tiles = gemm_nt_tile_count): a FragCtx for a fragment-view functor, an EpiCtx for a row-view one.
template <class Epi>
__device__ __forceinline__ auto make_epi_ctx(const GemmNTParams& p, int i, int n_tiles, int tile_step, int it, int col0, int ncols,
                                             float* scratch) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, nch = (ncols + 31) >> 5;
    const int tile = gemm_nt_tile_at(p, i);
    const int next_tile = i + 2 * tile_step < n_tiles ? gemm_nt_tile_at(p, i + 2 * tile_step) : -1;
    if constexpr (FragmentEpilogue<Epi>) {
        const int row0 = tile * p.rows_per_tile;
        return FragCtx{row0, min(p.rows_per_tile, p.M - row0), warp & 3, nch, col0, ncols, scratch, wg, it, next_tile};
    } else {
        EpiCtx c;
        c.tile = tile;
        c.r = 32 * (warp & 1) + lane;
        c.grow = tile * p.rows_per_tile + c.r;
        c.valid = (c.r < p.rows_per_tile) && (c.grow < p.M);
        c.col0 = col0;
        c.ncols = ncols;
        c.tid = threadIdx.x;
        c.wg = wg;
        c.wtid = threadIdx.x & 127;
        c.half = (warp >> 1) & 1;
        epi_chunk_range(ncols, c.half, c.ch0, c.ch1);
        c.rounds = (nch + 1) >> 1;
        c.scratch = scratch;
        c.it = it;
        c.next_tile = next_tile;
        return c;
    }
}

// Row-view epilogues that move whole 32-row x 32-column bf16 tiles cooperatively stage them per warp (SWIZZLE_64B layout:
// 16-byte chunk q of row r at r*64 + ((q ^ (r>>1)) & 3)*16, conflict-free for row-per-lane 16-byte accesses).  Row-per-thread
// stores of 32 rows sit in the LSU queue and stall the warps on their source registers.
constexpr int kTileStoreBufs = 2;                                  // staging tiles per warp (2 KB each)
constexpr int kTileStoreBytes = kEpiWarps * kTileStoreBufs * 2048 + 1024;  // + alignment slack

// ---------------------------------------------------------------------------------------------
// gemm_nt kernel: one CTA per (tile sequence, weight slice)
// ---------------------------------------------------------------------------------------------
// mbarrier protocol:
//   bfull     count 1 + tx of the resident weight slice    -> the consumers may start (not used when b_stream)
//   full[s]   count 1 + tx of one A box (+ its weight box when b_stream; the producer's expect_tx)
//   empty[s]  count 4: every warp of the warpgroup that consumes stage s arrives once its wgmmas on it have completed
// The producer fills the ring in the CTA's tile order (taps * k_chunks stages per tile); each warpgroup walks the ring past
// the other warpgroup's tiles.
// MMA turn (named barriers kBarTurn + w, 256 threads): warpgroup w waits on its barrier before issuing a tile (except the
// CTA's first tile) and, once all its wgmmas are issued, arrives on the other warpgroup's barrier if the CTA has a next tile.
// Every arrive therefore meets exactly one wait, and the tiles' MMAs run in the CTA's tile order.
// The MMAs of one tile with NCH chunks (a compile-time N keeps the wgmmas asynchronous): one wgmma group per ring stage, one
// group left in flight while the next stage is awaited; a stage is released once its group completed.
template <int NCH>
__device__ __forceinline__ void gemm_nt_mma_tile(float* acc, const GemmNTParams& p, uint64_t* full, uint64_t* empty, int& st,
                                                 uint32_t& ph, uint32_t a_s, uint32_t b_s, int b_region, int lane, int pass_bar) {
    // the first k-step overwrites the accumulators (scale_d = 0): start a fresh value here, so that the previous tile's
    // accumulators are dead once the epilogue has read them instead of occupying registers through the whole epilogue
#pragma unroll
    for (int i = 0; i < 16 * NCH; ++i) asm volatile("" : "=f"(acc[i]));
    int prev = -1;
    for (int s = 0; s < p.taps; ++s)
        for (int kc = 0; kc < p.k_chunks; ++kc) {
            mbar_wait(&full[st], ph, 104);
            const uint32_t a_st = a_s + st * p.stage_bytes;
            const uint32_t b_box = p.b_stream ? a_st + kAStageBytes : b_s + (s * p.k_chunks + kc) * b_region;
            const uint64_t da = make_sw128_desc(a_st, 16, 1024), db = make_sw128_desc(b_box, 16, 1024);
            const int first = (s | kc) == 0;
#pragma unroll
            for (int i = 0; i < 16 * NCH; ++i) wgmma_reg_fence(acc[i]);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)  // +32 bytes per k-step = +2 in the descriptor's >>4 address field
                Wgmma<32 * NCH, 0, 0>::mma(acc, da + 2 * k, db + 2 * k, (first && k == 0) ? 0 : 1);
            wgmma_commit();
            wgmma_wait<1>();  // the group of the previous stage has completed
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);  // this warp's reads of stage prev are complete
            }
            prev = st;
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
    if (pass_bar >= 0) named_bar_arrive(pass_bar, 2 * kWgThreads);  // the other warpgroup may issue its tile
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 16 * NCH; ++i) wgmma_reg_fence(acc[i]);
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
    float* xpose = reinterpret_cast<float*>(sA + p.stages * p.stage_bytes);  // row view only
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(xpose) + (FragmentEpilogue<Epi> ? 0 : kXposeBytes));
    uint64_t* full = bars;
    uint64_t* empty = bars + kMaxStages;
    uint64_t* bfull = bars + 2 * kMaxStages;
    float* scratch = reinterpret_cast<float*>(bars + 2 * kMaxStages + 8);

    const int slice = blockIdx.x % p.n_slices;
    const int tile0 = blockIdx.x / p.n_slices;
    const int tile_step = gridDim.x / p.n_slices;
    // tile0 .. n_tiles are list positions (tiles themselves without a list).  A CTA without a tile leaves before it issues the
    // weight-slice load or touches a barrier.
    const int n_tiles = gemm_nt_tile_count(p);
    if (tile0 >= n_tiles) return;
    const int col0 = slice * p.n_stride;
    const int ncols = min(p.n_stride, p.N - col0);
    const int tap_shift = p.tap_origin;
    // tuning counters: [0] producer waits for a free A stage, [1] the CTA's weight slice, [5] kernel; per consumer warpgroup w
    // at [8 + 4w]: +0 waits for its MMA turn, +1 MMA loops incl. waits for A data (turn waits excluded), +2 epilogue, +3 tiles
    long long* tmr = p.timing != nullptr ? p.timing + blockIdx.x * 16 : nullptr;
    const long long t_begin = tmr != nullptr ? clock64() : 0;

    if (warp == kEpiWarps && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 4);
        }
        mbar_init(bfull, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= kEpiWarps) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kNtProducerRegs));
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
        long long tw_empty = 0;
        for (int i = tile0; i < n_tiles; i += tile_step) {
            const int row0 = gemm_nt_tile_at(p, i) * p.rows_per_tile;
            for (int s = 0; s < p.taps; ++s)
                for (int kc = 0; kc < p.k_chunks; ++kc) {
                    const long long t = tmr != nullptr ? clock64() : 0;
                    mbar_wait(&empty[st], ph ^ 1, 101);
                    if (tmr != nullptr) tw_empty += clock64() - t;
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
        if (tmr != nullptr && lane == 0) tmr[0] = tw_empty;
    } else {
        // ===================== consumer warpgroups: whole tiles in turn, wgmma then the epilogue =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kNtConsumerRegs));
        const int wg = warp >> 2;
        const int nch = (ncols + 31) >> 5;
        const int rounds = (nch + 1) >> 1;
        const EpiInit ei{col0, ncols, static_cast<int>(threadIdx.x), scratch, tile0, n_tiles};
        epi.init(ei, tile_step);
        const uint32_t a_s = smem_u32(sA), b_s = smem_u32(sB);
        float acc[128];
        const RegAcc racc{acc, xpose + wg * (kXposeBytes / 4 / 2), rounds, nch, kBarWg + wg};
        if (!p.b_stream) mbar_wait(bfull, 0, 102);
        int st = 0;
        uint32_t ph = 0;
        const int tile_stages = p.taps * p.k_chunks;
        auto skip_tile = [&]() {  // the ring stages of the other warpgroup's tile
            st += tile_stages;
            while (st >= p.stages) { st -= p.stages; ph ^= 1; }
        };
        if (wg == 1) skip_tile();
        long long tw_turn = 0, tw_mma = 0, tw_epi = 0;
        int it = 0;
        for (int i = tile0 + wg * tile_step; i < n_tiles; i += 2 * tile_step, ++it) {
            long long t = tmr != nullptr ? clock64() : 0;
            if (i != tile0) named_bar_sync(kBarTurn + wg, 2 * kWgThreads);  // the other warpgroup has issued its tile
            if (tmr != nullptr) { const long long u = clock64(); tw_turn += u - t; t = u; }
            const int pass_bar = i + tile_step < n_tiles ? kBarTurn + (wg ^ 1) : -1;
            switch (nch) {
                case 1: gemm_nt_mma_tile<1>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
                case 2: gemm_nt_mma_tile<2>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
                case 3: gemm_nt_mma_tile<3>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
                case 4: gemm_nt_mma_tile<4>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
                case 5: gemm_nt_mma_tile<5>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
                case 6: gemm_nt_mma_tile<6>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
                case 7: gemm_nt_mma_tile<7>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
                default: gemm_nt_mma_tile<8>(acc, p, full, empty, st, ph, a_s, b_s, b_region, lane, pass_bar); break;
            }
            skip_tile();
            if (tmr != nullptr) { const long long u = clock64(); tw_mma += u - t; t = u; }
            const auto ctx = make_epi_ctx<Epi>(p, i, n_tiles, tile_step, it, col0, ncols, scratch);
            if constexpr (FragmentEpilogue<Epi>) epi.frag(acc, ctx);
            else epi(racc, ctx);
            if (tmr != nullptr) tw_epi += clock64() - t;
        }
        epi.finish(ei);
        if (tmr != nullptr && (threadIdx.x & 127) == 0) {
            long long* w = tmr + 8 + 4 * wg;
            w[0] = tw_turn; w[1] = tw_mma; w[2] = tw_epi; w[3] = it;
            if (wg == 0) {
                tmr[1] = slice;
                tmr[5] = clock64() - t_begin;
            }
        }
    }
}

// Debug backend (TRIAGE builds only -- `make TRIAGE=1`, -DNEWSREC_TRIAGE; the release library has no second backend and
// consults no environment switch on the launch path): plain SIMT accumulate + the SAME epilogue functors, with the same two
// warpgroups taking the CTA's tiles in turn.
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
    const int wg = threadIdx.x >> 7;
    for (int i = threadIdx.x; i < Epi::kScratchBytes / 4; i += kEpiThreads) scratch[i] = 0.f;
    __syncthreads();
    const int n_tiles = gemm_nt_tile_count(p);
    const EpiInit ei{col0, ncols, static_cast<int>(threadIdx.x), scratch, tile0, n_tiles};
    epi.init(ei, tile_step);
    int it = 0;
    for (int i = tile0 + wg * tile_step; i < n_tiles; i += 2 * tile_step, ++it) {
        const int tile = gemm_nt_tile_at(p, i);
        const auto c = make_epi_ctx<Epi>(p, i, n_tiles, tile_step, it, col0, ncols, scratch);
        if constexpr (FragmentEpilogue<Epi>) {  // the same fragment layout as the wgmma accumulators
            const int lane = threadIdx.x & 31;
            float acc[128];
            for (int j = 0; j < 4 * c.nch; ++j)
                for (int e = 0; e < 2; ++e)
                    for (int i = 0; i < 2; ++i)
                        acc[4 * j + 2 * e + i] = p.dbg_acc[(static_cast<size_t>(tile) * kTileM + 16 * c.wq + (lane >> 2) + 8 * e) * p.dbg_ld +
                                                           col0 + 8 * j + 2 * (lane & 3) + i];
            epi.frag(acc, c);
        } else {
            GlobalAcc acc{p.dbg_acc + (static_cast<size_t>(tile) * kTileM + c.r) * p.dbg_ld + col0, c.ch0, c.ch1};
            epi(acc, c);
        }
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
    int cluster_m;   // cluster shape over (m-tile, n-tile): the CTAs of one k-range that share an A chunk (same m-tile) or a
    int cluster_n;   // B chunk (same n-tile) receive it by one TMA multicast; 1 x 1 = no cluster
    int k_slices;
    int chunks_per_slice;  // 64-row chunks per CTA (without k_list)
    // null: every 64-row chunk of the Kr rows.  Otherwise the chunks to reduce over, written on the device before the launch
    // (GemmNTParams::tile_list layout); the k_slices ranges split them evenly
    const int* k_list;
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
// epi_smem_bytes = kEpiSmemBytes<Epi>; max_n_stride (0 = none) caps the slice width for epilogues whose staging
// grows with it.
int plan_gemm_nt(GemmNTPlan* plan, const void* A, int M, int lda, const void* B, int N, int ldb, int K, int taps,
                 int b_tap_rows, int rows_per_tile, int num_sms, int max_slices, int epi_smem_bytes, int max_n_stride);
bool debug_simt_gemm();
// Thread-block clusters of cluster_x x cluster_y CTAs of `func` that fit on the device at once (cached per function and shape).
int max_active_clusters(const void* func, int threads, size_t smem, int cluster_x, int cluster_y);

template <class Epi>
int launch_gemm_nt(const GemmNTPlan& plan, const Epi& epi, const void* A, int lda, const void* B, int ldb,
                   cudaStream_t stream) {
    if (plan.p.num_m_tiles <= 0) return 0;
#ifdef NEWSREC_TRIAGE
    if (debug_simt_gemm()) {
        GemmNTParams p = plan.p;
        const size_t ld = static_cast<size_t>(round_up(p.N, 32) + 32);
        float* acc = nullptr;
        NR_CHECK_CUDA(cudaMallocAsync(&acc, sizeof(float) * ld * p.num_m_tiles * kTileM, stream));
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

}  // namespace nr
