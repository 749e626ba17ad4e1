// Shared helpers for the sm_90a kernels of the ngp_pl hot path.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define NGP_WARP 32

// Every C-ABI entry point returns 0 on success, a cudaError_t (>0) on a CUDA failure,
// or NGP_EINVAL (<0) for an argument the op cannot honour. Nothing allocates.
#define NGP_EINVAL (-22)

// process-wide count of the kernel launches this library has issued (eager launches and launches recorded into a CUDA
// graph under capture alike; defined in network.cu, read through ngp_launch_count()). Host threads only.
extern unsigned long long g_ngp_launch_count;
#define NGP_COUNT_LAUNCHES(k) (__atomic_fetch_add(&g_ngp_launch_count, (unsigned long long)(k), __ATOMIC_RELAXED))

// Debugging aid (tools/step_timeline.py): once a trace buffer is installed with ngp_trace_set(), the training-step entry
// points enqueue a one-thread kernel after each of their kernels that appends {id, %globaltimer} to it -- recorded into
// CUDA graphs like any other launch, so install it BEFORE capturing. Off (nullptr) in normal operation.
extern unsigned long long* g_ngp_trace;
void ngp_trace_stamp(int id, cudaStream_t st);
__device__ __forceinline__ void trace_mark(unsigned long long* buf, int id) {  // what the stamp kernel does, from inside a kernel
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    const unsigned long long i = atomicAdd(&buf[0], 1ull);
    if (i < buf[1]) {
        buf[2 + 2 * i] = (unsigned long long)id;
        buf[3 + 2 * i] = t;
    }
}
#define NGP_TRACE(id, st)                                    \
    do {                                                     \
        if (g_ngp_trace) ngp_trace_stamp((id), (st));        \
    } while (0)

#define NGP_CHECK_LAUNCH()                                   \
    do {                                                     \
        NGP_COUNT_LAUNCHES(1);                               \
        cudaError_t _e = cudaGetLastError();                 \
        if (_e != cudaSuccess) return (int)_e;               \
    } while (0)

#define NGP_CUDA(call)                                       \
    do {                                                     \
        cudaError_t _e = (call);                             \
        if (_e != cudaSuccess) return (int)_e;               \
    } while (0)

static inline int ngp_div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Number of SMs of the current device (132 on H100 SXM); cached per process.
static inline int ngp_sm_count() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    }
    return sms;
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
// inclusive scans across the 32 lanes of a warp
__device__ __forceinline__ float warp_scan_add(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    return v;
}
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v *= u;
    }
    return v;
}

// L2 eviction-priority hints. The optimiser streams ~400 MB (params, moments, gradients) through the 50 MB L2 once per
// step; without hints that evicts the fp16 hash table (24 MB), the zeroed gradient table (49 MB) and the occupancy
// bitfield which the next step's kernels gather from / reduce into, and those kernels then run from DRAM.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ float4 ld_f4_hint(const float4* ptr, uint64_t policy) {
    float4 v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(ptr), "l"(policy));
    return v;
}
__device__ __forceinline__ void st_f4_hint(float4* ptr, float4 v, uint64_t policy) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(ptr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w),
                 "l"(policy)
                 : "memory");
}
__device__ __forceinline__ void st_u2_hint(uint2* ptr, uint2 v, uint64_t policy) {
    asm volatile("st.global.L2::cache_hint.v2.u32 [%0], {%1,%2}, %3;" ::"l"(ptr), "r"(v.x), "r"(v.y), "l"(policy) : "memory");
}

// 8-byte vector reduction (two fp32 adds in one L2 atomic transaction; sm_90+)
__device__ __forceinline__ void red_add_f32x2(float* addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// 16-byte vector reduction (four fp32 adds in one L2 atomic transaction; sm_90+), 16-byte aligned address
__device__ __forceinline__ void red_add_f32x4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_half2(uint32_t u) {
    __half2 h = *reinterpret_cast<__half2*>(&u);
    return __half22float2(h);
}
