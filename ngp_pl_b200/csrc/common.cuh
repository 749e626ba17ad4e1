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

// Programmatic dependent launch (sm_90). The training step is a serial chain of kernels on one stream; launched with
// ngp_launch_pdl(), a kernel may start while its immediate predecessor in the stream is still running (stream capture
// records the edge as a programmatic graph edge), so its launch latency and prologue hide under the predecessor's tail.
// pdl_wait() returns once the predecessor has completed and its writes are visible; pdl_trigger() lets the successor
// launch. A kernel launched without the attribute (any plain <<<>>> launch) returns from pdl_wait() at once.
// The rules that make a chain of such kernels safe:
//  - every thread of a kernel calls pdl_wait() exactly once, before it exits, and pdl_trigger() only after its own
//    pdl_wait(). Then, when a kernel starts, every kernel before its immediate predecessor has completed and its writes
//    are visible;
//  - before its pdl_wait(), a kernel reads nothing its immediate predecessor writes;
//  - before its pdl_wait(), a kernel writes nothing its immediate predecessor reads or writes.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t ngp_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                         Args&&... args) {
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Let Kernel use `bytes` (> 48 KB) of dynamic shared memory on the current device. The opt-in is a per-device function
// attribute and one process may drive several GPUs, so it is set once per device (device ordinals past 63: every call).
template <auto Kernel>
static inline cudaError_t ngp_smem_opt_in(int bytes) {
    static unsigned char set[64] = {0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const bool cached = dev >= 0 && dev < 64;
    if (cached && __atomic_load_n(&set[dev], __ATOMIC_ACQUIRE)) return cudaSuccess;
    e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && cached) __atomic_store_n(&set[dev], 1, __ATOMIC_RELEASE);
    return e;
}

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

// Whether the device can address p: device or managed memory, or (host_mapped_ok) mapped pinned host memory whose host
// pointer is its device pointer.
static inline bool ngp_dev_ptr(const void* p, bool host_mapped_ok) {
    if (!p) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();  // a failed query is not an error of the next launch
        return false;
    }
    if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) return true;
    return host_mapped_ok && a.type == cudaMemoryTypeHost && a.devicePointer == p;
}

// One camera ray (reference datasets/ray_utils.py:46-70): rays_d = direction @ R^T, rays_o = t, for the 3x4
// camera-to-world pose P = [R | t] (row-major). The batch assembly and the viewer's frames share this arithmetic, so their
// rays are bitwise equal for the same pose and direction.
__device__ __forceinline__ void pose_ray(const float* __restrict__ P, float dx, float dy, float dz, float* __restrict__ o,
                                         float* __restrict__ d) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        // d_k = sum_c dir_c * R[k][c]
        d[k] = fmaf(dz, P[4 * k + 2], fmaf(dy, P[4 * k + 1], dx * P[4 * k]));
        o[k] = P[4 * k + 3];
    }
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
