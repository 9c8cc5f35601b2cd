// Common device/host helpers for the sm_90a news-recommendation hot path.
// Raw PTX wrappers for mbarrier / TMA / wgmma -- no CUTLASS dependency.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "nr_wgmma.cuh"

namespace nr {

// ----------------------------------------------------------------------------------------------
// error plumbing (host)
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
#define NR_CHECK_CUDA(expr)                                                                   \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            nr::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return (int)_e;                                                                   \
        }                                                                                     \
    } while (0)
#define NR_REQUIRE(cond, ...)                \
    do {                                     \
        if (!(cond)) {                       \
            nr::set_error(__VA_ARGS__);      \
            return -1;                       \
        }                                    \
    } while (0)
#define NR_PROPAGATE(expr)          \
    do {                            \
        int _r = (expr);            \
        if (_r != 0) return _r;     \
    } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

// ----------------------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

// Device-side watchdog record: [0]=code, [1]=block, [2]=thread, [3]=aux.  Read by nr_device_error().
// Lives in the one translation unit that owns the mbarrier pipelines (gemm.cu defines NR_OWNS_WATCHDOG).
#ifdef NR_OWNS_WATCHDOG
__device__ int g_dev_error[4] = {0, 0, 0, 0};
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// try_wait with a suspend-time hint: the warp sleeps in hardware until the phase completes or `ns` nanoseconds pass.  Without
// the hint the instruction gives up after ~30 cycles and a waiting warp turns into a busy loop that competes for issue
// slots with the warps it is waiting for (ncu on the fused front end: 8 waiting warps per SM took most of the issue slots,
// tensor pipe 8 % active).
__device__ __forceinline__ bool mbar_try_wait_sleep(uint64_t* bar, uint32_t parity, uint32_t ns) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
        : "memory");
    return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread for a system-dependent time when the phase is not complete)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a mis-programmed pipeline traps after ~4 s instead of hanging the GPU.
#ifdef NR_OWNS_WATCHDOG
__device__ __noinline__ void mbar_timeout(int code, uint32_t aux) {
    g_dev_error[0] = code;
    g_dev_error[1] = blockIdx.x;
    g_dev_error[2] = threadIdx.x;
    g_dev_error[3] = (int)aux;
    __threadfence_system();
    asm volatile("trap;");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int code) {
    if (mbar_try_wait_sleep(bar, parity, 20000u)) return;
    uint64_t t0 = 0;
    while (!mbar_try_wait_sleep(bar, parity, 1000000u)) {  // every failed probe slept for up to 1 ms (or came back early: timed below)
        const uint64_t t = globaltimer_ns();
        if (t0 == 0) t0 = t;
        else if (t - t0 > 4000000000ull) mbar_timeout(code, parity);
    }
}
#endif

// ---- TMA (cp.async.bulk.tensor) -----------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// The same box landing at the same shared-memory offset in every CTA of cta_mask (bit r = cluster rank r); each receiver's
// mbarrier at bar's offset sees the complete_tx of its copy.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}

// ---- thread-block clusters ---------------------------------------------------------------------
// every thread of every CTA of the cluster; release / acquire: shared-memory writes (mbarrier inits included) before it are
// visible to the partners after it
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at bar's offset in the shared memory of cluster rank `rank` (this CTA's own included).  Release at
// CTA scope (the default) is what a consumer's "stage read" needs; .release.cluster would first wait for every earlier
// global write of the thread, the epilogue's reductions and stores included.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    asm volatile(
        "{\n\t.reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
        ::"r"(smem_u32(bar)), "r"(rank)
        : "memory");
}

// TMA store of one box from shared memory (bulk async-group completion)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_src), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
    tma_store_2d(m, smem_u32(smem_src), c0, c1);
}
// bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned) from shared to global memory (bulk async-group completion)
__device__ __forceinline__ void bulk_store_1d(void* gdst, uint32_t smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {  // at most N groups of this thread still reading shared memory
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// Explicit shared-space loads (the epilogue scratch is reached through a generic pointer; LD.E through the generic
// path is slower than LDS).  volatile keeps them ordered against the other asm statements, where they are placed by hand.
__device__ __forceinline__ float4 lds_f4(const float* p) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(smem_u32(p)));
    return v;
}
__device__ __forceinline__ float lds_f(const float* p) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(smem_u32(p)));
    return v;
}
__device__ __forceinline__ float2 lds_f2(const float* p) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(smem_u32(p)));
    return v;
}
__device__ __forceinline__ uint4 lds_u4(uint32_t saddr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr) : "memory");
    return v;
}
// Four 8x8 b16 matrices to shared memory: lanes 8m .. 8m+7 give the row addresses of matrix m, and register m of lane t holds
// row t/4, columns 2(t%4) and 2(t%4)+1 of matrix m -- the mma accumulator layout, packed to bf16 pairs.
__device__ __forceinline__ void stmatrix_x4(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
                 : "memory");
}
// 4-byte cp.async with zero fill when !pred (src must still be a valid address)
__device__ __forceinline__ void cp_async_f32(float* smem_dst, const float* gsrc, bool pred) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(pred ? 4 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// wgmma shared-memory matrix descriptor, SWIZZLE_128B:
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout = 1 (128-byte swizzle)
// K-major operand: rows of 128 bytes (64 bf16 of K), SBO = 1024 between 8-row groups.  MN-major operand: LBO = bytes between
// 64-element blocks along M / N, SBO = 1024 between 8-row groups along K.  A k-step of 16 elements adds 32 bytes (K-major)
// or 2048 bytes (MN-major) to the start address.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFFu);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

// ---- small math / packing ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
    return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
// tanh(x) = 1 - 2/(exp(2x)+1); ex2.approx + rcp.approx: abs error ~2e-7, saturates cleanly.
__device__ __forceinline__ float fast_tanh(float x) {
    const float e = exp2f(x * 2.8853900817779268f);  // exp(2x); -use_fast_math -> ex2.approx
    return 1.0f - __fdividef(2.0f, e + 1.0f);
}
// MUFU.TANH: one instruction, max relative error 2^-11 -- below the bf16 rounding of everything it feeds in the
// BACKWARD epilogues (the forward keeps fast_tanh: its scores are compared with the oracle at 1e-3).
__device__ __forceinline__ float tanh_approx(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float fast_sigmoid(float x) {
    return __fdividef(1.0f, 1.0f + exp2f(-x * 1.4426950408889634f));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// 32 values per lane -> lane l ends with the sum over lanes of v[l] (31 shuffles).
__device__ __forceinline__ float warp_transpose_sum32(float* v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int off = 16, n = 32; off >= 1; off >>= 1, n >>= 1) {
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < n / 2; ++i) {
            const float send = up ? v[i] : v[i + n / 2];
            const float keep = up ? v[i + n / 2] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
    return v[0];
}
__device__ __forceinline__ void red_add_f32(float* addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_v4_f32(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
                 : "memory");
}

// Counter-based dropout bits: (seed, element-group index) -> four 16-bit lanes (Dropout below draws its masks from them).
// Two chained 32-bit multiply-xorshift rounds (about half the instructions of the splitmix64 finaliser this replaced,
// which was >50 % of the instructions of the gather and of the dropout-carrying GEMM epilogues); the statistical tests
// (keep rate, scaling, train/eval mean) are the acceptance criterion for the mask quality.
__device__ __forceinline__ uint64_t dropout_bits4(uint64_t seed, uint64_t group) {
    const uint32_t g_lo = static_cast<uint32_t>(group), g_hi = static_cast<uint32_t>(group >> 32);
    uint32_t x = (g_lo ^ static_cast<uint32_t>(seed)) + g_hi * 0x85EBCA6Bu + static_cast<uint32_t>(seed >> 32) * 0x165667B1u;
    x *= 0x9E3779B1u;
    x ^= x >> 15;
    x *= 0x85EBCA77u;
    x ^= x >> 13;
    uint32_t y = x * 0xC2B2AE3Du + static_cast<uint32_t>(seed >> 32);
    y ^= y >> 16;
    y *= 0x27D4EB2Fu;
    y ^= y >> 15;
    return (static_cast<uint64_t>(y) << 32) | x;
}

// The library's dropout mask.  Element (row, col) of a matrix with pitch ld (a multiple of 4) is in group (row * ld + col) >> 2
// and is kept iff 16-bit lane col & 3 of dropout_bits4(seed, group) is >= thresh; a kept element is multiplied by scale.  The
// forward and the backward of a composite draw the same mask from the same (p, seed).  These members are the only code that
// tests a lane against thresh; the Python reference model of the kernels (the oracle) restates the rule.
struct Dropout {
    float p;          // 0 => off
    float scale;      // 1/(1-p); 1 when off
    uint32_t thresh;  // round(p * 65536)
    uint64_t seed;

    static Dropout make(float p, uint64_t seed) {
        return Dropout{p, p > 0.f ? 1.f / (1.f - p) : 1.f, static_cast<uint32_t>(p * 65536.0f + 0.5f), seed};
    }
    __device__ __forceinline__ bool active() const { return p > 0.f; }
    // multipliers of the aligned 4-column group at col4 of a row
    __device__ __forceinline__ void mask4(long long row, int ld, int col4, float* m) const {
        mask4_group((static_cast<uint64_t>(row) * ld + col4) >> 2, m);
    }
    // the same for a precomputed group index ((row * ld + col) >> 2; callers that walk a row keep row * ld / 4 in a register);
    // 32-bit field tests: the 64-bit shifts / compares of the straightforward form were a quarter of the instructions of the
    // dropout-carrying epilogues (ncu source page)
    __device__ __forceinline__ void mask4_group(uint64_t group, float* m) const {
        const uint64_t bits = dropout_bits4(seed, group);
        const uint32_t lo = static_cast<uint32_t>(bits), hi = static_cast<uint32_t>(bits >> 32);
        m[0] = ((lo & 0xffffu) >= thresh) ? scale : 0.f;
        m[1] = ((lo >> 16) >= thresh) ? scale : 0.f;
        m[2] = ((hi & 0xffffu) >= thresh) ? scale : 0.f;
        m[3] = ((hi >> 16) >= thresh) ? scale : 0.f;
    }
    // multipliers of element col (.x) and, for an even col, of its pair col + 1 (.y) of a row.  The lane is picked from the two
    // 32-bit halves by selects: indexing a float[4] at a run-time position would put the array in local memory.
    __device__ __forceinline__ float2 mask2(long long row, int ld, int col) const {
        const uint64_t bits = dropout_bits4(seed, (static_cast<uint64_t>(row) * ld + col) >> 2);
        const uint32_t w = (col & 2) ? static_cast<uint32_t>(bits >> 32) : static_cast<uint32_t>(bits);
        const uint32_t own = (col & 1) ? (w >> 16) : (w & 0xffffu);
        return make_float2(own >= thresh ? scale : 0.f, (w >> 16) >= thresh ? scale : 0.f);
    }
    // the same masks applied to one 32-column chunk of a wgmma fragment: y[4jj + 2e + i] is row[e], column col + 8jj +
    // 2 (lane % 4) + i.  The mask of (row, aligned 4-column group) is one hash; lanes 2k and 2k+1 hold columns 0-1 and 2-3 of
    // the same group in both rows: lane bit b hashes row e = b and passes the partner the 32-bit half it needs
    __device__ __forceinline__ void apply_frag(float* y, const long long* row, int ld, int col) const {
        const int lane = threadIdx.x & 31, b = lane & 1;
        const long long my_row = b ? row[1] : row[0];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int col4 = col + 8 * jj + 4 * ((lane >> 1) & 1);
            const uint64_t bits = dropout_bits4(seed, (static_cast<uint64_t>(my_row) * ld + col4) >> 2);
            const uint32_t lo = static_cast<uint32_t>(bits), hi = static_cast<uint32_t>(bits >> 32);
            const uint32_t own = b ? hi : lo, other = __shfl_xor_sync(0xffffffffu, b ? lo : hi, 1);
            const uint32_t wd[2] = {b ? other : own, b ? own : other};
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                y[4 * jj + 2 * e] *= ((wd[e] & 0xffffu) >= thresh) ? scale : 0.f;
                y[4 * jj + 2 * e + 1] *= ((wd[e] >> 16) >= thresh) ? scale : 0.f;
            }
        }
    }
};

#endif  // __CUDACC__

// ----------------------------------------------------------------------------------------------
// host: TMA tensor-map encoding through the driver entry point (no link-time libcuda dependency)
// ----------------------------------------------------------------------------------------------
// 2-D bf16 tensor [rows][cols] with row pitch ld (elements), box = [box_cols(<=64) x box_rows];
// swizzle_bytes = 128 (operand tiles, box_cols <= 64), 64 (epilogue store tiles, box_cols <= 32) or 0 (dense row-major
// box, rows of box_cols * 2 bytes, a multiple of 16).
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, int64_t rows, int64_t cols, int64_t ld_elems, int box_cols,
                      int box_rows, int swizzle_bytes = 128);
int make_tmap_bytes_2d(CUtensorMap* out, const void* base, int64_t rows, int64_t row_bytes, int64_t pitch_bytes, int box_bytes,
                       int box_rows);

}  // namespace nr
