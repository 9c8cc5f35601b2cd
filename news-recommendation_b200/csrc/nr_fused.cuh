// Device error record and bounded mbarrier wait of the translation units that keep their own watchdog record
// (gru_persist.cu, attn_title.cu).
#pragma once
#include "nr_common.cuh"

namespace nr {
namespace fused {

// ---- device error record + bounded waits of the fused kernels -------------------------------------------------------------
// every translation unit of this family names its own record (no relocatable device code): #define NR_WATCHDOG_SYMBOL first
#ifdef NR_WATCHDOG_SYMBOL
__device__ int NR_WATCHDOG_SYMBOL[4] = {0, 0, 0, 0};
static __device__ __noinline__ void f_timeout(int code, uint32_t aux) {
    NR_WATCHDOG_SYMBOL[0] = code;
    NR_WATCHDOG_SYMBOL[1] = blockIdx.x;
    NR_WATCHDOG_SYMBOL[2] = threadIdx.x;
    NR_WATCHDOG_SYMBOL[3] = static_cast<int>(aux);
    __threadfence_system();
    asm volatile("trap;");
}
__device__ __forceinline__ void f_wait(uint64_t* bar, uint32_t parity, int code) {
    if (mbar_try_wait_sleep(bar, parity, 20000u)) return;
    uint64_t t0 = 0;
    while (!mbar_try_wait_sleep(bar, parity, 1000000u)) {  // sleeps in hardware; wakes when the phase completes
        const uint64_t t = globaltimer_ns();
        if (t0 == 0) t0 = t;
        else if (t - t0 > 4000000000ull) f_timeout(code, parity);
    }
}
#endif

}  // namespace fused
}  // namespace nr
