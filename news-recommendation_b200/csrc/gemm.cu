// wgmma GEMM building blocks + their fused-epilogue instantiations.  See nr_gemm.cuh for the design.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#define NR_OWNS_WATCHDOG 1
#include "nr_epilogues.cuh"
#include "nr_ops.h"

namespace nr {

static_assert(kGemmTileRows == kTileM, "nr_ops.h and nr_gemm.cuh disagree on the gemm_nt tile height");
int read_gru_device_error(int* out4);
int g_launches = 0;

// ------------------------------------------------------------------------------------------------
// error string (thread local) + device watchdog record
// ------------------------------------------------------------------------------------------------
static thread_local char t_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}
const char* last_error() { return t_err; }
int read_device_error(int* out4) {
    const int rc = (int)cudaMemcpyFromSymbol(out4, g_dev_error, sizeof(int) * 4);
    if (rc != 0 || out4[0] != 0) return rc;
    return read_gru_device_error(out4);  // the persistent GRU kernel keeps its own record (gru_persist.cu)
}

// ------------------------------------------------------------------------------------------------
// live per-kernel timing
// ------------------------------------------------------------------------------------------------
struct ProfRec {
    std::string name;
    cudaEvent_t a, b;
};
static bool g_prof_on = false;
static std::string g_prof_ctx;
static std::vector<ProfRec> g_prof;
static std::vector<cudaEvent_t> g_prof_pool;
static cudaEvent_t prof_event() {
    cudaEvent_t e;
    if (!g_prof_pool.empty()) {
        e = g_prof_pool.back();
        g_prof_pool.pop_back();
    } else {
        cudaEventCreate(&e);
    }
    return e;
}
void prof_enable(int on) { g_prof_on = on != 0; }
void prof_context(const char* ctx) { g_prof_ctx = ctx; }
// NEWSREC_TRACE=1: print every launch and synchronise after it (pin-points a stuck or faulting kernel).
static int trace_on() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("NEWSREC_TRACE");
        v = (e != nullptr && e[0] == '1') ? 1 : 0;
    }
    return v;
}
ProfScope::ProfScope(const char* op, int a, int b, int c, cudaStream_t s) : idx(-1), stream(s) {
    if (trace_on()) {
        fprintf(stderr, "[nr] launch %s/%s[%d,%d,%d]\n", g_prof_ctx.c_str(), op, a, b, c);
        fflush(stderr);
    }
    if (!g_prof_on) return;
    char buf[160];
    snprintf(buf, sizeof(buf), "%s/%s[%d,%d,%d]", g_prof_ctx.c_str(), op, a, b, c);
    ProfRec r{buf, prof_event(), prof_event()};
    cudaEventRecord(r.a, s);
    idx = static_cast<int>(g_prof.size());
    g_prof.push_back(r);
}
ProfScope::~ProfScope() {
    if (idx >= 0) cudaEventRecord(g_prof[idx].b, stream);
    if (trace_on()) {
        const cudaError_t e = cudaStreamSynchronize(stream);
        fprintf(stderr, "[nr]   -> %s\n", cudaGetErrorString(e));
        fflush(stderr);
    }
}
int prof_report(char* buf, int cap) {
    std::map<std::string, std::pair<int, double>> agg;
    for (auto& r : g_prof) {
        float ms = 0.f;
        if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
            auto& e = agg[r.name];
            e.first += 1;
            e.second += ms;
        }
        g_prof_pool.push_back(r.a);
        g_prof_pool.push_back(r.b);
    }
    g_prof.clear();
    std::string out = "{";
    bool first = true;
    for (auto& kv : agg) {
        char line[256];
        snprintf(line, sizeof(line), "%s\"%s\": [%d, %.6f]", first ? "" : ", ", kv.first.c_str(), kv.second.first,
                 kv.second.second);
        out += line;
        first = false;
    }
    out += "}";
    if (static_cast<int>(out.size()) + 1 > cap) return -1;
    memcpy(buf, out.c_str(), out.size() + 1);
    return static_cast<int>(out.size());
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
            n = 0;
        if (const char* e = getenv("NEWSREC_NUM_SMS")) n = atoi(e);
    }
    return n;
}

#ifdef NEWSREC_TRIAGE
static int g_debug_simt = -1;
bool debug_simt_gemm() {
    if (g_debug_simt < 0) {
        const char* e = getenv("NEWSREC_DEBUG_SIMT_GEMM");
        g_debug_simt = (e != nullptr && e[0] == '1') ? 1 : 0;
    }
    return g_debug_simt == 1;
}
void set_debug_simt_gemm(int on) { g_debug_simt = on ? 1 : 0; }
int has_triage_backends() { return 1; }
#else
bool debug_simt_gemm() { return false; }
void set_debug_simt_gemm(int) {}
int has_triage_backends() { return 0; }
#endif
// tuning (tools/kbench.py): device buffer [slots][148][16]; every planned gemm_nt takes the next slot
static long long* g_gemm_timing = nullptr;
static int g_gemm_timing_slots = 0, g_gemm_timing_next = 0;
void set_debug_gemm_timing(void* dev_buf, int slots) {
    g_gemm_timing = static_cast<long long*>(dev_buf);
    g_gemm_timing_slots = slots;
    g_gemm_timing_next = 0;
}

// ------------------------------------------------------------------------------------------------
// TMA descriptor encoding via the driver entry point (resolved at run time: the library must load
// on a machine without libcuda so that the CPU-side symbol tests can dlopen it)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, int64_t rows, int64_t cols, int64_t ld_elems, int box_cols,
                      int box_rows, int swizzle_bytes) {
    EncodeTiledFn enc = get_encode();
    NR_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
    NR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base %p not 16B aligned", base);
    NR_REQUIRE((ld_elems * 2) % 16 == 0, "TMA row pitch %lld elements is not a multiple of 16 bytes", (long long)ld_elems);
    NR_REQUIRE(((swizzle_bytes == 128 || swizzle_bytes == 64) ? box_cols * 2 <= swizzle_bytes
                                                               : (swizzle_bytes == 0 && (box_cols * 2) % 16 == 0 && box_cols <= 256)) &&
                   box_rows <= 256 && box_rows >= 1,
               "bad TMA box %d x %d (swizzle %d)", box_cols, box_rows, swizzle_bytes);
    NR_REQUIRE(rows >= 1 && cols >= 1, "empty tensor for TMA (%lld x %lld)", (long long)rows, (long long)cols);
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld_elems) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE),
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    NR_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld cols=%lld ld=%lld box=%dx%d)",
               (int)r, (long long)rows, (long long)cols, (long long)ld_elems, box_cols, box_rows);
    return 0;
}

// Untyped 2-D tensor map: rows of `row_bytes` valid bytes at pitch `pitch_bytes`, moved as 8-byte elements (so that a box
// can be up to 2 KB wide), box = box_bytes x box_rows, no swizzle.  box_bytes may exceed row_bytes: the tail is zero
// filled on loads and dropped on stores (it lets the caller choose a bank-conflict-free row pitch in shared memory).
int make_tmap_bytes_2d(CUtensorMap* out, const void* base, int64_t rows, int64_t row_bytes, int64_t pitch_bytes, int box_bytes,
                       int box_rows) {
    EncodeTiledFn enc = get_encode();
    NR_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
    NR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && pitch_bytes % 16 == 0 && row_bytes % 8 == 0 && row_bytes >= 8,
               "TMA bytes map: base %p / pitch %lld / row %lld misaligned", base, (long long)pitch_bytes, (long long)row_bytes);
    NR_REQUIRE(box_bytes % 16 == 0 && box_bytes >= 16 && box_bytes <= 2048 && box_rows >= 1 && box_rows <= 256 && rows >= 1,
               "TMA bytes map: bad box %d B x %d", box_bytes, box_rows);
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(row_bytes / 8), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch_bytes)};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(box_bytes / 8), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    NR_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (bytes) failed with CUresult %d (rows=%lld row=%lld pitch=%lld box=%dx%d)", (int)r,
               (long long)rows, (long long)row_bytes, (long long)pitch_bytes, box_bytes, box_rows);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// gemm_nt planning
// ------------------------------------------------------------------------------------------------
int plan_gemm_nt(GemmNTPlan* plan, const void* A, int M, int lda, const void* B, int N, int ldb, int K, int taps,
                 int b_tap_rows, int rows_per_tile, int sms, int max_slices, int epi_smem_bytes, int max_n_stride) {
    NR_REQUIRE(M >= 0 && N >= 1 && K >= 1 && taps >= 1 && taps <= 4 && rows_per_tile >= 1 && rows_per_tile <= kTileM,
               "plan_gemm_nt: bad shape M=%d N=%d K=%d taps=%d rpt=%d", M, N, K, taps, rows_per_tile);
    NR_REQUIRE(sms > 0, "no CUDA device (SM count unknown)");
    GemmNTParams& p = plan->p;
    memset(&p, 0, sizeof(p));
    p.M = M;
    p.rows_per_tile = rows_per_tile;
    p.num_m_tiles = ceil_div(M, rows_per_tile);
    p.N = N;
    p.K = K;
    p.k_chunks = ceil_div(K, kChunkK);
    p.taps = taps;
    p.tap_origin = taps / 2;
    p.b_tap_rows = b_tap_rows;
#ifdef NEWSREC_TRIAGE
    static const int dbg_flags = [] { const char* v = getenv("NEWSREC_GEMM_DBG"); return v != nullptr ? atoi(v) : 0; }();
    p.dbg_flags = dbg_flags;
#endif
    if (g_gemm_timing != nullptr && g_gemm_timing_next < g_gemm_timing_slots) {
        p.timing = g_gemm_timing + static_cast<size_t>(g_gemm_timing_next) * 148 * 16;
        fprintf(stderr, "[nr] gemm timing slot %d: M=%d N=%d K=%d taps=%d\n", g_gemm_timing_next, M, N, K, taps);
        ++g_gemm_timing_next;
    }
    const int fixed = 1024 + round_up(epi_smem_bytes, 16) + 512;
    int slices = 1;
    long bbytes = 0;
    for (;; ++slices) {
        NR_REQUIRE(slices <= 64, "plan_gemm_nt: cannot fit weight slice (N=%d K=%d taps=%d)", N, K, taps);
        p.n_stride = round_up(ceil_div(N, slices), 16);  // 32-byte aligned slice starts (STG.256 epilogues)
        // whole 32-column chunks of resident weight rows: a warpgroup's wgmma covers its chunks entirely (rows past the
        // slice are the next slice's weights or TMA zero fill, never uninitialised shared memory)
        p.n_box = round_up(std::min(p.n_stride, N), 32);
        if (p.n_box > 256 || (max_n_stride > 0 && p.n_stride > max_n_stride)) continue;
        bbytes = static_cast<long>(taps) * p.k_chunks * p.n_box * 128;
        // a ring of 6 stages (48 KB) holds more than one tile of K <= 320 ahead of the MMAs
        if (bbytes + 6L * kAStageBytes + fixed <= kSmemLimit) break;
        // epilogues that reduce over the whole output row need ONE slice, and slices of <= 64 columns re-read A too often:
        // accept a shallower A ring, or else stream the weight boxes with the A tiles instead of keeping them resident
        if (slices == max_slices || p.n_box <= 64) {
            if (bbytes + 4L * kAStageBytes + fixed > kSmemLimit) {
                p.b_stream = 1;
                bbytes = 0;
            }
            break;
        }
    }
    p.n_slices = ceil_div(N, p.n_stride);
    p.stage_bytes = kAStageBytes + (p.b_stream ? p.n_box * 128 : 0);
    p.stages = static_cast<int>(std::min<long>(kMaxStages, (kSmemLimit - fixed - bbytes) / p.stage_bytes));
    NR_REQUIRE(p.stages >= 2, "plan_gemm_nt: only %d pipeline stages fit", p.stages);
    plan->smem = static_cast<size_t>(bbytes) + static_cast<size_t>(p.stages) * p.stage_bytes + fixed;
    // a group = n_slices CTAs working on the same 64-row tiles
    const int groups = std::max(1, std::min(sms / p.n_slices, p.num_m_tiles));
    plan->grid = groups * p.n_slices;
    if (p.num_m_tiles == 0) return 0;
    NR_PROPAGATE(make_tmap_bf16_2d(&plan->tmA, A, M, K, lda, kChunkK, kTileM));
    const int64_t brows = (taps > 1) ? static_cast<int64_t>(taps) * b_tap_rows : N;
    NR_PROPAGATE(make_tmap_bf16_2d(&plan->tmB, B, brows, K, ldb, kChunkK, p.n_box));
    return 0;
}

#ifdef NEWSREC_TRIAGE
// Debug backend accumulate: thread = one output column of one M tile (slow, obviously correct).
__global__ void gemm_nt_simt_acc_kernel(const __nv_bfloat16* A, int lda, const __nv_bfloat16* B, int ldb,
                                        GemmNTParams p) {
    const int n = blockIdx.x * 128 + threadIdx.x;
    const int tile = blockIdx.y;
    if (n >= p.dbg_ld) return;
    const int shift = p.tap_origin;
    for (int r = 0; r < kTileM; ++r) {
        float acc = 0.f;
        if (n < p.N) {
            for (int s = 0; s < p.taps; ++s) {
                const long long row = static_cast<long long>(tile) * p.rows_per_tile + r + s - shift;
                if (row < 0 || row >= p.M) continue;
                const __nv_bfloat16* a = A + row * lda;
                const __nv_bfloat16* b = B + static_cast<long long>(s * p.b_tap_rows + n) * ldb;
                for (int k = 0; k < p.K; ++k) acc = fmaf(__bfloat162float(a[k]), __bfloat162float(b[k]), acc);
            }
        }
        p.dbg_acc[(static_cast<size_t>(tile) * kTileM + r) * p.dbg_ld + n] = acc;
    }
}

#endif  // NEWSREC_TRIAGE

// ------------------------------------------------------------------------------------------------
// gemm_tn kernel: CTA = (128 output rows, <= 256 output columns, a range of 64-row k-chunks).  Warpgroup h owns output rows
// [64h, 64h + 64) and accumulates all NT columns in registers (MN-major operands straight from the TMA boxes); the result
// is added to D with vector reductions.
// ------------------------------------------------------------------------------------------------
template <int NT>
__global__ void __launch_bounds__(kTnThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmTNParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int kBoxes = NT / 64;
    constexpr int stage_bytes = (2 + kBoxes) * 8192;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes);
    uint64_t* full = bars;
    uint64_t* empty = bars + kMaxStages;

    const int mt = blockIdx.x, nt = blockIdx.y, ks = blockIdx.z;  // a cluster spans (m-tile, n-tile) pairs of one k-range
    // with a chunk list the k-ranges split the listed chunks evenly (the count is known on the device only)
    const int total_chunks = p.k_list != nullptr ? p.k_list[0] : (p.Kr + 63) >> 6;
    const int per_slice = p.k_list != nullptr ? (total_chunks + p.k_slices - 1) / p.k_slices : p.chunks_per_slice;
    const int chunk0 = ks * per_slice;
    const int n_my = max(0, min(per_slice, total_chunks - chunk0));
    const int n0 = nt * NT;                       // first output column of this CTA
    const int ncol = min(NT, p.Nb - n0);
    // cluster rank cx + cluster_m * cy; the A chunk of this m-tile goes to the ranks of column cx, the B chunk of this n-tile to
    // those of row cy.  Every CTA issues its share of both by multicast, so a stage may be refilled only once the consumers of
    // all those ranks have released it: the empty barriers count the warps of the row and the column.
    const bool clustered = p.cluster_m * p.cluster_n > 1;
    const int cx = mt % p.cluster_m, cy = nt % p.cluster_n;
    uint32_t a_mask = 0, b_mask = 0;
    for (int j = 0; j < p.cluster_n; ++j) a_mask |= 1u << (cx + p.cluster_m * j);
    for (int i = 0; i < p.cluster_m; ++i) b_mask |= 1u << (i + p.cluster_m * cy);

    if (warp == kEpiWarps && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8 * (p.cluster_m + p.cluster_n - 1));
        }
        fence_barrier_init();
    }
    if (clustered) cluster_sync();  // the partners' barriers exist before the first multicast or remote arrive
    else __syncthreads();
    if (n_my == 0) return;  // the whole cluster: its CTAs share the k-range

    if (warp >= kEpiWarps) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
        if (!clustered && warp != kEpiWarps) return;
    }
    if (warp == kEpiWarps) {
        // producer loop is warp-uniform, one elected lane issues
        int st = 0;
        uint32_t ph = 0;
        for (int c = 0; c < n_my; ++c) {
            const int k0 = (p.k_list != nullptr ? p.k_list[1 + chunk0 + c] : chunk0 + c) * 64;
            mbar_wait(&empty[st], ph ^ 1, clustered ? 203 : 201);
            if (elect_one()) {
                mbar_arrive_expect_tx(&full[st], static_cast<uint32_t>(stage_bytes));
                uint8_t* sa = smem + st * stage_bytes;
                uint8_t* sb = sa + 2 * 8192;
                if (!clustered) {
                    tma_load_2d(sa, &tmA, &full[st], mt * 128, k0);
                    tma_load_2d(sa + 8192, &tmA, &full[st], mt * 128 + 64, k0);
#pragma unroll
                    for (int j = 0; j < kBoxes; ++j)
                        tma_load_2d(sb + j * 8192, &tmB, &full[st], p.b_col0 + n0 + j * 64, k0 + p.b_row_shift);
                } else {  // box b of the A chunk from rank (cx, b % cluster_n), box j of the B chunk from rank (j % cluster_m, cy)
#pragma unroll
                    for (int b = 0; b < 2; ++b)
                        if (b % p.cluster_n == cy)
                            tma_load_2d_multicast(sa + b * 8192, &tmA, &full[st], mt * 128 + 64 * b, k0, static_cast<uint16_t>(a_mask));
#pragma unroll
                    for (int j = 0; j < kBoxes; ++j)
                        if (j % p.cluster_m == cx)
                            tma_load_2d_multicast(sb + j * 8192, &tmB, &full[st], p.b_col0 + n0 + j * 64, k0 + p.b_row_shift,
                                                  static_cast<uint16_t>(b_mask));
                }
            }
            __syncwarp();
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
    } else if (warp < kEpiWarps) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
        const int h = warp >> 2;
        float acc[NT / 2];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
        int st = 0;
        uint32_t ph = 0;
        for (int c = 0; c < n_my; ++c) {
            mbar_wait(&full[st], ph, 202);
            const uint32_t sa = smem_u32(smem + st * stage_bytes) + h * 8192;
            const uint32_t sb = smem_u32(smem + st * stage_bytes) + 2 * 8192;
            const uint64_t da = make_sw128_desc(sa, 8192, 1024);
            const uint64_t db = make_sw128_desc(sb, 8192, 1024);
#pragma unroll
            for (int i = 0; i < NT / 2; ++i) wgmma_reg_fence(acc[i]);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)  // +2048 bytes per k-step = +128 in the descriptor's >>4 address field
                Wgmma<NT, 1, 1>::mma(acc, da + 128 * k, db + 128 * k, (c | k) ? 1 : 0);
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < NT / 2; ++i) wgmma_reg_fence(acc[i]);
            __syncwarp();
            if (lane == 0) {
                if (!clustered) {
                    mbar_arrive(&empty[st]);
                } else {
                    for (uint32_t m = a_mask | b_mask; m != 0; m &= m - 1) mbar_arrive_cluster(&empty[st], __ffs(m) - 1);
                }
            }
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
        // fragment: acc[4j + 2e + i] = row 16 * (warp % 4) + lane / 4 + 8e, column 8j + 2 * (lane % 4) + i
        const bool vec2 = (p.ldd & 1) == 0 && (reinterpret_cast<uintptr_t>(p.D) & 7) == 0;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int grow = mt * 128 + 64 * h + 16 * (warp & 3) + (lane >> 2) + 8 * e;
            if (grow >= p.Ma) continue;
            float* drow = p.D + static_cast<size_t>(grow) * p.ldd + n0;
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
                const int col = 8 * j + 2 * (lane & 3);
                const float v0 = acc[4 * j + 2 * e], v1 = acc[4 * j + 2 * e + 1];
                if (vec2 && col + 2 <= ncol) {
                    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(drow + col), "f"(v0), "f"(v1) : "memory");
                } else {
                    if (col < ncol) red_add_f32(drow + col, v0);
                    if (col + 1 < ncol) red_add_f32(drow + col + 1, v1);
                }
            }
        }
    }
    // no CTA leaves while a partner may still arrive on its barriers or multicast into its ring (the idle producer warps stay)
    if (clustered) cluster_sync();
}

#ifdef NEWSREC_TRIAGE
__global__ void gemm_tn_simt_kernel(const __nv_bfloat16* A, int lda, const __nv_bfloat16* B, int ldb, int b_rows,
                                    GemmTNParams p) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int m = blockIdx.y;
    if (n >= p.Nb || m >= p.Ma) return;
    float acc = 0.f;
    for (int k = 0; k < p.Kr; ++k) {
        const long long br = static_cast<long long>(k) + p.b_row_shift;
        if (br < 0 || br >= b_rows) continue;
        acc = fmaf(__bfloat162float(A[static_cast<size_t>(k) * lda + m]),
                   __bfloat162float(B[static_cast<size_t>(br) * ldb + p.b_col0 + n]), acc);
    }
    atomicAdd(p.D + static_cast<size_t>(m) * p.ldd + n, acc);
}
#endif

// SMs the split-K weight-gradient GEMM leaves free (set by a data-parallel caller): the all-reduce of the embedding gradient
// is issued on a side stream right before this GEMM, and NCCL's channel CTAs need SMs to run on -- with every SM holding a
// 200 KB gemm_tn CTA the "overlapped" reduction simply waited for the GEMM to finish (2 GPUs: +0.27 ms per step, unchanged).
static int g_comm_reserved_sms = 0;
void set_comm_reserved_sms(int n) { g_comm_reserved_sms = n < 0 ? 0 : n; }

int max_active_clusters(const void* func, int threads, size_t smem, int cluster_x, int cluster_y) {
    static std::map<std::tuple<const void*, int, size_t, int, int>, int> cache;
    const auto key = std::make_tuple(func, threads, smem, cluster_x, cluster_y);
    const auto it = cache.find(key);
    if (it != cache.end()) return it->second;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster_x;
    attr[0].val.clusterDim.y = cluster_y;
    attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(cluster_x, cluster_y);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, func, &cfg) != cudaSuccess) n = 0;
    cache[key] = n;
    return n;
}

// Splits the reduction over k-ranges so that the grid fills the GPU once (with clusters: as many as fit at once), then launches.
template <int NT>
static int launch_gemm_tn_kernel(int sms, int total_chunks, size_t smem, const CUtensorMap& tmA, const CUtensorMap& tmB, GemmTNParams p,
                                 cudaStream_t stream) {
    static bool attr_set = false;  // per instantiation
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(gemm_tn_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
        attr_set = true;
    }
    const int tiles = p.m_tiles * p.n_tiles, csize = p.cluster_m * p.cluster_n;
    int k_slices = std::max(1, std::min(sms / tiles, total_chunks));
    if (csize > 1) {
        const int fit = max_active_clusters(reinterpret_cast<const void*>(gemm_tn_kernel<NT>), kTnThreads, smem, p.cluster_m, p.cluster_n);
        NR_REQUIRE(fit >= 1, "gemm_tn: no %d x %d cluster with %zu bytes of shared memory fits", p.cluster_m, p.cluster_n, smem);
        k_slices = std::max(1, std::min(k_slices, fit / (tiles / csize)));
    }
    p.chunks_per_slice = ceil_div(total_chunks, k_slices);
    p.k_slices = ceil_div(total_chunks, p.chunks_per_slice);
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = p.cluster_m;
    attr[0].val.clusterDim.y = p.cluster_n;
    attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(p.m_tiles, p.n_tiles, p.k_slices);
    cfg.blockDim = dim3(kTnThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = csize > 1 ? 1 : 0;
    NR_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemm_tn_kernel<NT>, tmA, tmB, p));
    return 0;
}

int gemm_tn_accumulate(const void* A, int Kr, int Ma, int lda, const void* B, int b_rows, int b_cols, int ldb,
                       int b_col0, int Nb, int b_row_shift, float* D, int ldd, cudaStream_t stream, const int* k_list) {
    NR_REQUIRE(Nb >= 1 && Nb <= 512 && Ma >= 1 && Kr >= 0, "gemm_tn: bad shape Kr=%d Ma=%d Nb=%d", Kr, Ma, Nb);
    if (Kr == 0) return 0;
    GemmTNParams p;
    memset(&p, 0, sizeof(p));
    p.Kr = Kr;
    p.Ma = Ma;
    p.Nb = Nb;
    p.b_col0 = b_col0;
    p.b_row_shift = b_row_shift;
    p.D = D;
    p.ldd = ldd;
    p.k_list = k_list;
    ProfScope ps("gemm_tn", Kr, Ma, Nb, stream);
#ifdef NEWSREC_TRIAGE
    if (debug_simt_gemm()) {
        dim3 g(ceil_div(Nb, 64), Ma);
        gemm_tn_simt_kernel<<<g, 64, 0, stream>>>(static_cast<const __nv_bfloat16*>(A), lda,
                                                  static_cast<const __nv_bfloat16*>(B), ldb, b_rows, p);
        ++g_launches;
        NR_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
#endif
    NR_REQUIRE(num_sms() > 0, "no CUDA device");
    const int sms = std::max(num_sms() / 2, num_sms() - g_comm_reserved_sms);
    p.m_tiles = ceil_div(Ma, 128);
    // output columns per CTA: <= 256 (the accumulators of one warpgroup), in whole 64-column boxes
    p.n_tiles = ceil_div(Nb, 256);
    const int nt_cols = round_up(ceil_div(Nb, p.n_tiles), 64);
    const int total_chunks = ceil_div(Kr, 64);
    // a cluster of 2 along each tile dimension that divides: the two CTAs share the chunk of the other operand
    p.cluster_m = p.m_tiles % 2 == 0 ? 2 : 1;
    p.cluster_n = p.n_tiles % 2 == 0 ? 2 : 1;
    p.n_boxes = nt_cols / 64;
    const int stage_bytes = (2 + p.n_boxes) * 8192;
    p.stages = std::min(kMaxStages, (kSmemLimit - 1024 - 512) / stage_bytes);
    NR_REQUIRE(p.stages >= 2, "gemm_tn: stage of %d bytes does not double-buffer", stage_bytes);
    p.stages = std::min(p.stages, 6);
    CUtensorMap tmA, tmB;
    NR_PROPAGATE(make_tmap_bf16_2d(&tmA, A, Kr, Ma, lda, 64, 64));
    NR_PROPAGATE(make_tmap_bf16_2d(&tmB, B, b_rows, b_cols, ldb, 64, 64));
    const size_t smem = static_cast<size_t>(p.stages) * stage_bytes + 1024 + 512;
    switch (p.n_boxes) {
        case 1: NR_PROPAGATE(launch_gemm_tn_kernel<64>(sms, total_chunks, smem, tmA, tmB, p, stream)); break;
        case 2: NR_PROPAGATE(launch_gemm_tn_kernel<128>(sms, total_chunks, smem, tmA, tmB, p, stream)); break;
        case 3: NR_PROPAGATE(launch_gemm_tn_kernel<192>(sms, total_chunks, smem, tmA, tmB, p, stream)); break;
        default: NR_PROPAGATE(launch_gemm_tn_kernel<256>(sms, total_chunks, smem, tmA, tmB, p, stream)); break;
    }
    ++g_launches;
    return 0;
}

int gemm_weight_grad(const void* dY, int M, int N, int ld_dy, const void* X, int K, int ldx, float* dW_ext, cudaStream_t stream, int x_row_shift,
                     const int* k_list) {
    for (int c0 = 0; c0 < K + 1; c0 += 512)
        NR_PROPAGATE(gemm_tn_accumulate(dY, M, N, ld_dy, X, M, K + 1, ldx, c0, std::min(512, K + 1 - c0), x_row_shift, dW_ext + c0, ldx, stream,
                                        k_list));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// epilogue instantiations
// ------------------------------------------------------------------------------------------------
static RowMap to_rm(const RowMapCfg& c) { return RowMap{c.seg_in, c.in_off, c.seg_len, c.seg_out, c.out_off}; }

// the chunk path of EpiStore emits the low plane by whole 32-column chunks of a weight slice: no chunk may straddle lo_col0
static bool lo_plane_chunk_aligned(const GemmNTParams& p, int lo_col0) {
    for (int sl = 0; sl < p.n_slices; ++sl) {
        const int c0 = sl * p.n_stride;
        if (c0 < lo_col0 && lo_col0 < c0 + p.n_stride && (lo_col0 - c0) % 32 != 0) return false;
    }
    return true;
}
bool gemm_store_lo_supported(int N, int K, int lo_col0) {
    GemmNTPlan plan;  // the weight slicing depends on N and K only: plan an empty problem
    if (plan_gemm_nt(&plan, nullptr, 0, K, nullptr, N, K, K, 1, 0, kTileM, 1, 0, kEpiSmemBytes<EpiStore>, 0) != 0) return false;
    return lo_col0 >= 0 && lo_col0 < N && lo_plane_chunk_aligned(plan.p, lo_col0);
}

// the operands' tap origin (GemmOperands::tap_origin) over the planner's centred default
static int apply_tap_origin(GemmNTPlan& plan, const GemmOperands& g) {
    if (g.tap_origin < 0) return 0;
    NR_REQUIRE(g.tap_origin < g.taps, "gemm: tap origin %d outside %d taps", g.tap_origin, g.taps);
    plan.p.tap_origin = g.tap_origin;
    return 0;
}

int gemm_store(const GemmOperands& g, const StoreCfg& c, cudaStream_t stream) {
    if (g.M == 0) return 0;
    const int M = g.M, N = g.N, rows_per_tile = std::min(c.rows_per_tile, kTileM);  // every row is owned by exactly one tile
    GemmNTPlan plan;
    NR_PROPAGATE(plan_gemm_nt(&plan, g.A, M, g.lda, g.W, N, g.ldw, g.K, g.taps, g.w_tap_rows, rows_per_tile, num_sms(), 0,
                              kEpiSmemBytes<EpiStore>, 0));
    NR_PROPAGATE(apply_tap_origin(plan, g));
    NR_REQUIRE(c.tile_list == nullptr || rows_per_tile == kTileM, "gemm_store: a tile list needs whole 64-row tiles");
    plan.p.tile_list = c.tile_list;
    NR_REQUIRE(c.out_bf16 ? (c.ld_out % 8 == 0) : (c.ld_out % 4 == 0), "gemm_store: output pitch %d breaks vector stores", c.ld_out);
    // the ones column is written by slice 0's CTA with plain stores after its chunk loop: only past the result columns (a chunk
    // of another slice, or one of its own TMA stores still in flight, would race with it) and only inside the row's pitch
    NR_REQUIRE(c.ones_col < 0 || (c.out_bf16 && c.ones_col >= N && c.ones_col < c.ld_out),
               "gemm_store: the ones column needs a bf16 output and N <= ones_col < ld_out (N=%d ones_col=%d ld=%d)", N, c.ones_col,
               c.ld_out);
    NR_REQUIRE(c.ones_zero_upto <= c.ld_out, "gemm_store: zeroed columns up to %d run past the output pitch %d", c.ones_zero_upto,
               c.ld_out);
    EpiStore e;
    memset(&e, 0, sizeof(e));
    e.use_tma = (c.out_bf16 && c.rm.seg_in == 0 && rows_per_tile == kTileM && N >= 32) ? 1 : 0;
    if (e.use_tma) NR_PROPAGATE(make_tmap_bf16_2d(&e.tm_out, c.out, M, N, c.ld_out, 32, 16, 64));
    e.lo_col0 = -1;
    NR_REQUIRE(!c.accumulate || !c.out_bf16, "gemm_store: accumulation needs an fp32 output");
    e.accumulate = c.accumulate;
    if (c.lo_out != nullptr) {
        const int lo_col0 = c.lo_col0, ld_lo = c.ld_lo;
        NR_REQUIRE(c.out_bf16 && lo_col0 >= 0 && lo_col0 < N && ld_lo % 8 == 0 && ld_lo >= N - lo_col0 && (e.use_tma || lo_col0 % 8 == 0),
                   "gemm_store: the low plane needs bf16 output and aligned columns (N=%d lo_col0=%d ld_lo=%d)", N, lo_col0, ld_lo);
        NR_REQUIRE(lo_plane_chunk_aligned(plan.p, lo_col0), "gemm_store: low-plane start %d is not chunk aligned in its weight slice (N=%d)",
                   lo_col0, N);
        if (e.use_tma) NR_PROPAGATE(make_tmap_bf16_2d(&e.tm_lo, c.lo_out, M, N - lo_col0, ld_lo, 32, 16, 64));
        e.lo_col0 = lo_col0;
        e.lo_out = static_cast<__nv_bfloat16*>(c.lo_out);
        e.ld_lo = ld_lo;
    }
    e.out = c.out;
    e.ld = c.ld_out;
    e.out_bf16 = c.out_bf16;
    e.bias = c.bias;
    e.relu = c.relu;
    NR_REQUIRE(!(c.relu && c.tanh), "gemm_store: one activation at a time");
    e.act_tanh = c.tanh;
    if (c.dtanh_src != nullptr)
        NR_REQUIRE(c.dtanh_ld % 2 == 0 && (reinterpret_cast<uintptr_t>(c.dtanh_src) & 3) == 0,
                   "gemm_store: the tanh-backward source needs 4-byte aligned column pairs (ld=%d)", c.dtanh_ld);
    e.dtanh_src = static_cast<const __nv_bfloat16*>(c.dtanh_src);
    e.dtanh_ld = c.dtanh_ld;
    e.N = N;
    e.rm = to_rm(c.rm);
    e.drop = Dropout::make(c.drop.p, c.drop.seed);
    e.ones_col = c.ones_col;
    e.ones_cols_zero_upto = c.ones_zero_upto;
#ifdef NEWSREC_TRIAGE
    static const int dbg_skip = [] { const char* v = getenv("NEWSREC_EPI_DBG"); return v != nullptr && v[0] == '1' ? 1 : 0; }();
    e.dbg_skip = dbg_skip;
#endif
    g_launches += debug_simt_gemm() ? 2 : 1;
    ProfScope ps("gemm_store", M, N, g.K * g.taps, stream);
    return launch_gemm_nt(plan, e, g.A, g.lda, g.W, g.ldw, stream);
}

int gemm_additive_pool(const void* X, int M, int lda, int D, const void* Wa, int q, int ldw, const float* ba,
                       const float* qv, int seg_len, float* out, int ldo, float* w_out, cudaStream_t stream, const void* X_lo) {
    // the shape is checked before the empty case: seg_len = 0 makes M = n_seg * seg_len = 0 for any n_seg, and the segments'
    // outputs would be left unwritten without an error
    NR_REQUIRE(seg_len >= 1 && seg_len <= kTileM && M % seg_len == 0, "additive_pool: M=%d seg_len=%d", M, seg_len);
    NR_REQUIRE(q >= 1 && q <= 256 && (D % 2) == 0 && (ldo % 2) == 0, "additive_pool: q=%d D=%d ldo=%d unsupported", q, D, ldo);
    if (M == 0) return 0;
    const int rpt = (kTileM / seg_len) * seg_len;
    GemmNTPlan plan;
    NR_PROPAGATE(plan_gemm_nt(&plan, X, M, lda, Wa, q, ldw, D, 1, 0, rpt, num_sms(), 1, kEpiSmemBytes<EpiPool>, 0));
    NR_REQUIRE(plan.p.n_slices == 1, "additive_pool: the query dimension must fit one weight slice (q=%d D=%d)", q, D);
    EpiPool e;
    e.bias = ba;
    e.qv = qv;
    e.X = static_cast<const __nv_bfloat16*>(X);
    e.X_lo = static_cast<const __nv_bfloat16*>(X_lo);
    e.lda = lda;
    e.D = D;
    e.seg_len = seg_len;
    e.rows_per_tile = rpt;
    e.M = M;
    e.out = out;
    e.ldo = ldo;
    e.w_out = w_out;
    g_launches += debug_simt_gemm() ? 2 : 1;
    ProfScope ps("gemm_additive_pool", M, q, D, stream);
    return launch_gemm_nt(plan, e, X, lda, Wa, ldw, stream);
}

// The weight slicing of a plan depends on N, K, taps and the caps only: the shape checks below plan an empty problem, so that
// nr_additive_attention_bwd can run them before its first launch.
int additive_dpre_check(int q, int D, int ld_dpre) {
    NR_REQUIRE(q >= 1 && q <= 256 && ld_dpre % 8 == 0 && ld_dpre >= round_up(q, 8), "additive_dpre: q=%d ld=%d", q, ld_dpre);
    GemmNTPlan plan;
    NR_PROPAGATE(plan_gemm_nt(&plan, nullptr, 0, D, nullptr, q, D, D, 1, 0, kTileM, 1, 1, kEpiSmemBytes<EpiDPre>, 0));
    NR_REQUIRE(plan.p.n_slices == 1, "additive_dpre: q=%d D=%d does not fit one weight slice", q, D);
    return 0;
}

int gemm_additive_dpre(const void* X, int M, int lda, int D, const void* Wa, int q, int ldw, const float* ba,
                       const float* qv, const float* dscore, void* dpre, int ld_dpre, float* dqv,
                       cudaStream_t stream) {
    if (M == 0) return 0;
    NR_PROPAGATE(additive_dpre_check(q, D, ld_dpre));
    GemmNTPlan plan;
    NR_PROPAGATE(plan_gemm_nt(&plan, X, M, lda, Wa, q, ldw, D, 1, 0, kTileM, num_sms(), 1, kEpiSmemBytes<EpiDPre>, 0));
    EpiDPre e;
    memset(&e, 0, sizeof(e));
    e.use_tma = q >= 32 ? 1 : 0;
    if (e.use_tma) NR_PROPAGATE(make_tmap_bf16_2d(&e.tm_out, dpre, M, ld_dpre, ld_dpre, 32, 16, 64));
    e.bias = ba;
    e.qv = qv;
    e.dscore = dscore;
    e.dpre = static_cast<__nv_bfloat16*>(dpre);
    e.ld = ld_dpre;
    e.dqv = dqv;
    g_launches += debug_simt_gemm() ? 2 : 1;
    ProfScope ps("gemm_additive_dpre", M, q, D, stream);
    return launch_gemm_nt(plan, e, X, lda, Wa, ldw, stream);
}

// identity rows, no mask and at least one whole 32-column chunk: the fragment view; otherwise the row view
static bool pool_dinput_frag(const GemmOperands& g, const PoolDInputCfg& c) {
    return c.rm.seg_in == 0 && c.relu_src == nullptr && !c.zero_pad_rows && g.N >= 32;
}
// the epilogue stages the dOut rows of every segment a tile touches (<= 64 / seg_len + 2): cap the slice width so that they fit
static int pool_dinput_max_stride(int seg_len) { return (DOutStage::kStageFloats / (kTileM / seg_len + 2)) & ~15; }

int pool_dinput_check(const GemmOperands& g, const PoolDInputCfg& c) {
    const int seg_len = c.seg_len;
    NR_REQUIRE(seg_len >= 1, "pool_dinput: seg_len=%d", seg_len);
    const int max_stride = pool_dinput_max_stride(seg_len);
    NR_REQUIRE(max_stride >= 16, "pool_dinput: seg_len=%d needs %d staged segments per tile", seg_len, kTileM / seg_len + 2);
    NR_REQUIRE(c.ld_dx % 8 == 0, "pool_dinput: ld_dx=%d", c.ld_dx);
    GemmNTPlan plan;
    return plan_gemm_nt(&plan, nullptr, 0, g.lda, nullptr, g.N, g.ldw, g.K, g.taps, g.w_tap_rows, kTileM, 1, 0,
                        pool_dinput_frag(g, c) ? kEpiSmemBytes<EpiDPoolInFrag> : kEpiSmemBytes<EpiDPoolIn>, max_stride);
}

int gemm_pool_dinput(const GemmOperands& g, const PoolDInputCfg& c, cudaStream_t stream) {
    const int M = g.M, D = g.N, seg_len = c.seg_len;
    if (M == 0) return 0;
    NR_PROPAGATE(pool_dinput_check(g, c));
    const int max_stride = pool_dinput_max_stride(seg_len);
    GemmNTPlan plan;
    if (pool_dinput_frag(g, c)) {
        NR_PROPAGATE(plan_gemm_nt(&plan, g.A, M, g.lda, g.W, D, g.ldw, g.K, g.taps, g.w_tap_rows, kTileM, num_sms(), 0,
                                  kEpiSmemBytes<EpiDPoolInFrag>, max_stride));
        EpiDPoolInFrag e{.w = c.w, .dout = c.dout, .ldo = c.ldo, .seg_len = seg_len, .dx = static_cast<__nv_bfloat16*>(c.dx), .ld = c.ld_dx,
                         .N = D, .drop = Dropout::make(c.drop.p, c.drop.seed), .M = M};
        NR_PROPAGATE(make_tmap_bf16_2d(&e.tm_out, c.dx, M, D, c.ld_dx, 32, 16, 64));
        g_launches += debug_simt_gemm() ? 2 : 1;
        ProfScope ps("gemm_pool_dinput", M, D, g.K, stream);
        return launch_gemm_nt(plan, e, g.A, g.lda, g.W, g.ldw, stream);
    }
    NR_PROPAGATE(plan_gemm_nt(&plan, g.A, M, g.lda, g.W, D, g.ldw, g.K, g.taps, g.w_tap_rows, kTileM, num_sms(), 0, kEpiSmemBytes<EpiDPoolIn>,
                              max_stride));
    EpiDPoolIn e{.w = c.w, .dout = c.dout, .ldo = c.ldo,
                 .seg_len = seg_len, .dx = static_cast<__nv_bfloat16*>(c.dx), .ld = c.ld_dx, .N = D, .rm = to_rm(c.rm),
                 .zero_pad_rows = c.zero_pad_rows, .drop = Dropout::make(c.drop.p, c.drop.seed), .relu_src = static_cast<const __nv_bfloat16*>(c.relu_src),
                 .relu_ld = c.relu_ld, .M = M};
    g_launches += debug_simt_gemm() ? 2 : 1;
    ProfScope ps("gemm_pool_dinput", M, D, g.K, stream);
    return launch_gemm_nt(plan, e, g.A, g.lda, g.W, g.ldw, stream);
}

constexpr int kLiveTilesThreads = 256;
// The last block of a tile-flagging kernel to finish (ticket) compacts flags[0 .. num_tiles) in ascending tile order into
// list[0] = count, list[1 ..] = the flagged tiles.  Every block calls it after writing its own flags.
__device__ void compact_live_tiles(const int* flags, int num_tiles, unsigned* ticket, int* list) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __shared__ bool last;
    __shared__ int warp_sums[kLiveTilesThreads / 32];
    __threadfence();  // this block's flags are visible before its ticket
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    // thread i compacts the run of tiles [i * per, i * per + per): count, block-wide exclusive scan, then write
    const int per = (num_tiles + kLiveTilesThreads - 1) / kLiveTilesThreads;
    const int b = min(num_tiles, static_cast<int>(threadIdx.x) * per), e = min(num_tiles, b + per);
    int n = 0;
    for (int t = b; t < e; ++t) n += __ldcg(flags + t);
    int incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    int pos = incl - n;
    for (int w = 0; w < warp; ++w) pos += warp_sums[w];
    for (int t = b; t < e; ++t)
        if (__ldcg(flags + t)) list[1 + pos++] = t;
    if (threadIdx.x == kLiveTilesThreads - 1) list[0] = pos;  // the last run ends at the total
}

// The tiles of the embedding-gradient GEMM that scatter something: tile t (rows [64t, 64t + 64) of M) is live when one of its
// rows maps through rm to a token whose id is in [1, V) -- EpiScatter's own test, so a dead tile would add nothing.  Padded
// histories make runs of all-padding tiles (about 40 % of the NRMS batch), whose A loads and MMAs the scatter then skips.
// Each warp flags whole tiles; compact_live_tiles lists them (the layout of GemmNTParams::tile_list).
__global__ void __launch_bounds__(kLiveTilesThreads)
scatter_live_tiles_kernel(const long long* ids, int V, RowMap rm, int M, int num_tiles, int* flags, unsigned* ticket, int* list) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = kLiveTilesThreads / 32;
    for (int t = blockIdx.x * warps + warp; t < num_tiles; t += gridDim.x * warps) {
        bool live = false;
#pragma unroll
        for (int k = 0; k < kTileM / 32; ++k) {
            const int grow = t * kTileM + 32 * k + lane;
            long long trow;
            int tt;
            if (grow < M && rm.map(grow, trow, tt)) {
                const long long id = ids[trow];
                live = live || (id >= 1 && id < V);
            }
        }
        live = __any_sync(0xffffffffu, live);
        if (lane == 0) flags[t] = live ? 1 : 0;
    }
    compact_live_tiles(flags, num_tiles, ticket, list);
}

// ------------------------------------------------------------------------------------------------
// padding titles of the news encoder's forward (PaddingTitles in nr_ops.h).  A warp owns a 64-row tile and classifies every
// title that has a row in it (a title across a tile edge is classified by both tiles, the same way); the tile whose rows
// include a title's first row writes its flag.
// ------------------------------------------------------------------------------------------------
struct PaddingJob {
    const long long* ids;
    int n_seq, T, d, M, num_tiles;
    const uint32_t* row0;  // bf16 pairs: row 0 of the table
    const float* bqkv;     // non-null: also write the shared padding tile
    int sec, ld3;
    PaddingTitles out;
    unsigned* ticket;
};

// whether the first d columns of a bf16 row are nonzero (any block thread may ask; every thread of the block must)
__device__ __forceinline__ bool block_row_nonzero(const uint32_t* row, int d) {
    bool nz = false;
    for (int i = threadIdx.x; i < d / 2; i += blockDim.x) nz = nz || (row[i] & 0x7fff7fffu) != 0;
    return __syncthreads_or(nz) != 0;
}

// Q|K|V of a zero row: what the projection's store epilogue writes for it, bf16(0 + b) (and with vlo, bf16(y - bf16(y)))
__device__ __forceinline__ void write_padding_qkv(const float* bqkv, int T, int sec, int ld3, void* qkv_out, void* vlo_out) {
    const int n3 = 3 * sec;
    auto* qkv = static_cast<__nv_bfloat16*>(qkv_out);
    auto* vlo = static_cast<__nv_bfloat16*>(vlo_out);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < T * ld3; i += gridDim.x * blockDim.x) {
        const int c = i % ld3, r = i / ld3;
        const float y = c < n3 ? bqkv[c] : 0.f;
        const __nv_bfloat16 h = __float2bfloat16_rn(y);
        qkv[i] = h;
        if (vlo != nullptr && c >= 2 * sec && c < n3) vlo[r * sec + c - 2 * sec] = __float2bfloat16_rn(y - __bfloat162float(h));
    }
}

__global__ void __launch_bounds__(kLiveTilesThreads) padding_titles_kernel(const PaddingJob j) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = kLiveTilesThreads / 32;
    const bool row0_nonzero = block_row_nonzero(j.row0, j.d);  // one verdict for every title
    if (j.bqkv != nullptr) write_padding_qkv(j.bqkv, j.T, j.sec, j.ld3, j.out.qkv, j.out.v_lo);
    for (int t = blockIdx.x * warps + warp; t < j.num_tiles; t += gridDim.x * warps) {
        const int r0 = t * kTileM, r1 = min(j.M, r0 + kTileM);
        bool live = false;
        for (int s = r0 / j.T; s * j.T < r1; ++s) {
            const long long id = lane < j.T ? j.ids[static_cast<long long>(s) * j.T + lane] : 0;
            const bool pad = __all_sync(0xffffffffu, id == 0) && !row0_nonzero;
            live = live || !pad;
            if (lane == 0 && s * j.T >= r0) j.out.pad[s] = pad ? 1 : 0;
        }
        if (lane == 0) j.out.tile_flags[t] = live ? 1 : 0;
    }
    compact_live_tiles(j.out.tile_flags, j.num_tiles, j.ticket, j.out.live);
}

int padding_titles(const long long* ids, long long n_seq, int T, int d, const void* table, int ld_table, const float* bqkv, int sec,
                   int ld3, PaddingTitles* out, cudaStream_t stream) {
    NR_REQUIRE(T >= 1 && T <= 32 && d % 2 == 0 && ld_table % 8 == 0 && n_seq * T < (1ll << 31), "padding_titles: T=%d d=%d ld=%d", T,
               d, ld_table);
    const int M = static_cast<int>(n_seq * T), num_tiles = ceil_div(M, kTileM);
    // pad flags | tile flags | ticket | live list | shared Q|K|V tile | its V low plane; stream-ordered, freed by the caller
    const size_t pad_b = round_up(static_cast<int>(n_seq), 16), head_b = round_up(static_cast<int>(pad_b) + 4 * (2 * num_tiles + 2), 128);
    const size_t qkv_b = bqkv ? round_up(T * ld3 * 2, 128) : 0, vlo_b = bqkv ? static_cast<size_t>(T) * sec * 2 : 0;
    char* buf = nullptr;
    NR_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&buf), head_b + qkv_b + vlo_b, stream));
    out->base = buf;
    out->pad = reinterpret_cast<unsigned char*>(buf);
    out->tile_flags = reinterpret_cast<int*>(buf + pad_b);
    unsigned* ticket = reinterpret_cast<unsigned*>(out->tile_flags + num_tiles);
    out->live = out->tile_flags + num_tiles + 1;
    out->qkv = bqkv ? buf + head_b : nullptr;
    out->v_lo = bqkv ? static_cast<char*>(out->qkv) + qkv_b : nullptr;
    if (n_seq == 0) return 0;
    NR_CHECK_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned), stream));
    const PaddingJob j{.ids = ids, .n_seq = static_cast<int>(n_seq), .T = T, .d = d, .M = M, .num_tiles = num_tiles,
                       .row0 = static_cast<const uint32_t*>(table), .bqkv = bqkv, .sec = sec, .ld3 = ld3, .out = *out, .ticket = ticket};
    ProfScope ps("padding_titles", M, num_tiles, 0, stream);
    const int blocks = std::max(1, std::min(4 * num_sms(), ceil_div(num_tiles, kLiveTilesThreads / 32)));
    padding_titles_kernel<<<blocks, kLiveTilesThreads, 0, stream>>>(j);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

void free_padding_titles(PaddingTitles& pt, cudaStream_t stream) {
    if (pt.base != nullptr) cudaFreeAsync(pt.base, stream);
    pt = PaddingTitles{};
}

// ------------------------------------------------------------------------------------------------
// live tokens of the news encoder's backward (LiveTokens in nr_ops.h).  Block b of both kernels owns the titles
// [32 b, 32 b + 32); one warp classifies or compacts one title at a time.
//   classify: live mask, padding flag and live count of every title, the block's total; the last block to finish (ticket)
//             scans the block totals into block bases and writes M' and the tile count.  Also the shared padding Q|K|V
//             tile and the tile list body.
//   compact:  the block's per-title offsets (a block scan of its counts on top of its base), the compact -> token index,
//             the compact copy of the live X rows, and the zero tail rows [M', round_up(M', 64)).
// ------------------------------------------------------------------------------------------------
constexpr int kLiveTitlesPerBlock = 32;  // four titles per warp: about 900 blocks for a bench batch

struct LiveJob {
    const long long* ids;
    int n_seq, T, d, M, V, n_blocks;
    const uint32_t* row0;  // bf16 pairs: row 0 of the table, or null (the verdict from X)
    const float* bqkv;
    int sec, ld3, ldx;
    const uint4* X;        // bf16 rows of pitch ldx (16-byte pieces)
    uint4* Xc;
    uint4* dqkv_c;
    int* counts;           // [n_seq] live tokens per title
    int* block_base;       // [n_blocks] live tokens of the titles before the block
    unsigned* ticket;
    LiveTokens out;
};

__global__ void __launch_bounds__(kLiveTilesThreads) live_classify_kernel(const LiveJob j) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = kLiveTilesThreads / 32;
    const bool all_live = j.row0 != nullptr && block_row_nonzero(j.row0, j.d);
    write_padding_qkv(j.bqkv, j.T, j.sec, j.ld3, j.out.qkv, nullptr);
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
    for (int i = gtid; i < (j.M + kTileM - 1) / kTileM; i += nthreads) j.out.tiles[1 + i] = i;
    const int px = j.ldx / 8;  // 16-byte pieces per row of X
    const int s0 = blockIdx.x * kLiveTitlesPerBlock, s1 = min(j.n_seq, s0 + kLiveTitlesPerBlock);
    int total = 0;  // lane 0: the live tokens of this warp's titles
    for (int s = s0 + warp; s < s1; s += warps) {
        const long long id = lane < j.T ? j.ids[static_cast<long long>(s) * j.T + lane] : 0;
        uint32_t mask = __ballot_sync(0xffffffffu, lane < j.T && (all_live || (id >= 1 && id < j.V)));
        if (j.row0 == nullptr) {  // no table: a token whose gathered row is nonzero below column d is live as well
            for (uint32_t cand = ((j.T == 32 ? 0u : 1u << j.T) - 1u) & ~mask; cand != 0; cand &= cand - 1) {
                const int r = __ffs(cand) - 1;
                const uint4* x = j.X + (static_cast<long long>(s) * j.T + r) * px;
                uint32_t nz = 0;
                for (int c = lane; c < px; c += 32) {
                    const uint4 v = __ldg(x + c);
                    const int n = min(8, max(0, j.d - 8 * c));  // columns of this piece below d
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int k = 0; k < 4; ++k) nz |= w[k] & (2 * k + 1 < n ? 0x7fff7fffu : 2 * k < n ? 0x00007fffu : 0u);
                }
                if (__any_sync(0xffffffffu, nz != 0)) mask |= 1u << r;
            }
        }
        if (lane == 0) {
            j.out.mask[s] = mask;
            j.out.pad[s] = mask == 0 ? 1 : 0;
            j.counts[s] = __popc(mask);
            total += __popc(mask);
        }
    }
    __shared__ int warp_tot[kLiveTilesThreads / 32];
    __shared__ bool last;
    if (lane == 0) warp_tot[warp] = total;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < warps; ++w) t += warp_tot[w];
        j.block_base[blockIdx.x] = t;  // the block's total until the last block turns the totals into bases
        __threadfence();               // the total and this block's counts are visible before its ticket
        last = atomicAdd(j.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // exclusive scan of the block totals, kLiveTilesThreads at a time with a running carry
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int b0 = 0; b0 < j.n_blocks; b0 += kLiveTilesThreads) {
        const int b = b0 + threadIdx.x;
        const int v = b < j.n_blocks ? __ldcg(j.block_base + b) : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        int base = carry;
        for (int w = 0; w < warp; ++w) base += warp_tot[w];
        if (b < j.n_blocks) j.block_base[b] = base + incl - v;
        __syncthreads();
        if (threadIdx.x == kLiveTilesThreads - 1) carry = base + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        j.out.offset[j.n_seq] = carry;
        j.out.tiles[0] = (carry + kTileM - 1) / kTileM;
    }
}

__global__ void __launch_bounds__(kLiveTilesThreads) live_compact_kernel(const LiveJob j) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = kLiveTilesThreads / 32;
    const int s0 = blockIdx.x * kLiveTitlesPerBlock, s1 = min(j.n_seq, s0 + kLiveTitlesPerBlock);
    // offsets of the block's titles: lane t of warp 0 scans title s0 + t
    static_assert(kLiveTitlesPerBlock == 32, "one warp scans the block's titles");
    __shared__ int off[kLiveTitlesPerBlock];
    if (warp == 0) {
        const int v = s0 + lane < s1 ? j.counts[s0 + lane] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        off[lane] = j.block_base[blockIdx.x] + incl - v;
        if (s0 + lane < s1) j.out.offset[s0 + lane] = off[lane];
    }
    __syncthreads();
    // the tail rows [M', round_up(M', 64)) below M: no token, zero X and dQ|dK|dV rows (the last block)
    const int px = j.ldx / 8, p3 = j.ld3 / 8;  // 16-byte pieces per row
    if (blockIdx.x == gridDim.x - 1) {
        const int m_live = j.out.offset[j.n_seq];
        const int tail_end = min(j.M, (m_live + kTileM - 1) / kTileM * kTileM);
        for (int r = m_live + threadIdx.x; r < tail_end; r += blockDim.x) j.out.index[r] = -1;
        for (int i = threadIdx.x; i < (tail_end - m_live) * px; i += blockDim.x)
            j.Xc[static_cast<long long>(m_live) * px + i] = make_uint4(0, 0, 0, 0);
        for (int i = threadIdx.x; i < (tail_end - m_live) * p3; i += blockDim.x)
            j.dqkv_c[static_cast<long long>(m_live) * p3 + i] = make_uint4(0, 0, 0, 0);
    }
    // a warp per title: the index entries, then every 16-byte piece of the title's live rows spread over the lanes
    __shared__ int src_row[kLiveTilesThreads / 32][32];
    for (int s = s0 + warp; s < s1; s += warps) {
        const uint32_t mask = j.out.mask[s];
        const int dst = off[s - s0], n_live = __popc(mask);
        const int rank = __popc(mask & ((1u << lane) - 1u));
        if (lane < j.T && ((mask >> lane) & 1u)) {
            j.out.index[dst + rank] = s * j.T + lane;
            src_row[warp][rank] = s * j.T + lane;
        }
        __syncwarp();
        const uint4* X = j.X;
        uint4* Xc = j.Xc + static_cast<long long>(dst) * px;
#pragma unroll 4
        for (int i = lane; i < n_live * px; i += 32) {
            const int k = i / px, c = i - k * px;
            Xc[i] = __ldg(X + static_cast<long long>(src_row[warp][k]) * px + c);
        }
        __syncwarp();
    }
}

// bytes of the LiveTokens buffers of a call (live_tokens carves them from `buf`)
long long live_tokens_bytes(long long n_seq, int T, int ld3) {
    const long long n = n_seq, M = n_seq * T, nb = (n + kLiveTitlesPerBlock - 1) / kLiveTitlesPerBlock;
    WorkspaceLayout l{nullptr};
    l.take<unsigned char>(n);           // pad
    l.take<uint32_t>(n);                // mask
    l.take<int>(n);                     // counts
    l.take<int>(n + 1);                 // offset
    l.take<int>(M);                     // index
    l.take<int>(M / kTileM + 2);        // tiles
    l.take<int>(nb + 1);                // block bases | ticket
    l.take<__nv_bfloat16>(static_cast<long long>(T) * ld3);  // shared Q|K|V tile
    return l.bytes();
}

int live_tokens(const long long* ids, long long n_seq, int T, int d, const void* table, int ld_table, int V, const float* bqkv,
                int sec, int ld3, const void* X, int ldx, void* Xc, void* dqkv_c, void* buf, long long buf_bytes, LiveTokens* out,
                cudaStream_t stream) {
    NR_REQUIRE(ids && bqkv && X && Xc && dqkv_c && buf, "live_tokens: null operand");
    NR_REQUIRE(T >= 1 && T <= 32 && d % 2 == 0 && ld_table % 8 == 0 && ldx % 8 == 0 && ld3 % 8 == 0 && V >= 1 && n_seq * T < (1ll << 31),
               "live_tokens: T=%d d=%d ld_table=%d ldx=%d ld3=%d V=%d", T, d, ld_table, ldx, ld3, V);
    const auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    NR_REQUIRE(a16(X) && a16(Xc) && a16(dqkv_c) && a16(buf), "live_tokens: rows not 16-byte aligned");
    NR_REQUIRE(buf_bytes >= live_tokens_bytes(n_seq, T, ld3), "live_tokens: buffer too small (%lld bytes)", buf_bytes);
    const int n = static_cast<int>(n_seq), M = n * T, nb = ceil_div(n, kLiveTitlesPerBlock);
    WorkspaceLayout l{static_cast<char*>(buf)};
    out->pad = l.take<unsigned char>(n);
    out->mask = l.take<uint32_t>(n);
    int* counts = l.take<int>(n);
    out->offset = l.take<int>(n + 1);
    out->index = l.take<int>(M);
    out->tiles = l.take<int>(M / kTileM + 2);
    int* block_base = l.take<int>(nb + 1);
    out->qkv = l.take<__nv_bfloat16>(static_cast<long long>(T) * ld3);
    if (n == 0) return 0;
    unsigned* ticket = reinterpret_cast<unsigned*>(block_base + nb);
    NR_CHECK_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned), stream));
    const LiveJob j{.ids = ids, .n_seq = n, .T = T, .d = d, .M = M, .V = V, .n_blocks = nb, .row0 = static_cast<const uint32_t*>(table),
                    .bqkv = bqkv, .sec = sec, .ld3 = ld3, .ldx = ldx, .X = static_cast<const uint4*>(X), .Xc = static_cast<uint4*>(Xc),
                    .dqkv_c = static_cast<uint4*>(dqkv_c), .counts = counts, .block_base = block_base, .ticket = ticket, .out = *out};
    ProfScope ps("live_tokens", M, n, 0, stream);
    live_classify_kernel<<<nb, kLiveTilesThreads, 0, stream>>>(j);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    live_compact_kernel<<<nb, kLiveTilesThreads, 0, stream>>>(j);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int gemm_scatter_emb(const GemmOperands& g, const ScatterEmbCfg& c, cudaStream_t stream) {
    if (g.M == 0) return 0;
    NR_REQUIRE(g.N % 4 == 0 && c.V >= 1, "scatter_emb: N=%d V=%d", g.N, c.V);
    GemmNTPlan plan;  // every row is computed independently: whole tiles
    NR_PROPAGATE(plan_gemm_nt(&plan, g.A, g.M, g.lda, g.W, g.N, g.ldw, g.K, g.taps, g.w_tap_rows, kTileM, num_sms(), 0,
                              kEpiSmemBytes<EpiScatter>, 0));
    NR_PROPAGATE(apply_tap_origin(plan, g));
    const EpiScatter e{.ids = c.ids, .demb = c.demb, .V = c.V, .D = g.N, .rm = to_rm(c.rm), .drop = Dropout::make(c.drop.p, c.drop.seed),
                       .drop_ld = c.drop_ld, .rows = c.rows};
    NR_REQUIRE(c.rows == nullptr || c.rm.seg_in == 0, "scatter_emb: compact rows need the identity row map");
    if (c.tile_list != nullptr) {  // the caller knows the tiles with a live token
        plan.p.tile_list = c.tile_list;
        g_launches += debug_simt_gemm() ? 2 : 1;
        ProfScope ps("gemm_scatter_emb", g.M, g.N, g.K * g.taps, stream);
        return launch_gemm_nt(plan, e, g.A, g.lda, g.W, g.ldw, stream);
    }
    const int num_tiles = plan.p.num_m_tiles;
    // [0, num_tiles) flags | ticket | list (count + tiles); stream-ordered, so the buffer lives exactly as long as the two launches
    int* buf = nullptr;
    NR_CHECK_CUDA(cudaMallocAsync(&buf, sizeof(int) * (2 * static_cast<size_t>(num_tiles) + 2), stream));
    unsigned* ticket = reinterpret_cast<unsigned*>(buf + num_tiles);
    int* list = buf + num_tiles + 1;
    NR_CHECK_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned), stream));
    {
        ProfScope ps("scatter_live_tiles", g.M, num_tiles, 0, stream);
        const int blocks = std::max(1, std::min(4 * num_sms(), ceil_div(num_tiles, kLiveTilesThreads / 32)));
        scatter_live_tiles_kernel<<<blocks, kLiveTilesThreads, 0, stream>>>(c.ids, c.V, e.rm, g.M, num_tiles, buf, ticket, list);
        NR_CHECK_CUDA(cudaGetLastError());
        ++g_launches;
    }
    plan.p.tile_list = list;
    g_launches += debug_simt_gemm() ? 2 : 1;
    int rc;
    {
        ProfScope ps("gemm_scatter_emb", g.M, g.N, g.K * g.taps, stream);
        rc = launch_gemm_nt(plan, e, g.A, g.lda, g.W, g.ldw, stream);
    }
    NR_CHECK_CUDA(cudaFreeAsync(buf, stream));
    return rc;
}

}  // namespace nr
