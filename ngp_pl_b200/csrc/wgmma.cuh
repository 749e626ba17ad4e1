// Hopper (sm_90a) warpgroup MMA building blocks, hand-written PTX: shared-memory matrix descriptors, wgmma.mma_async with
// the fp32 accumulator in the registers of one warpgroup (4 warps), commit / wait of wgmma groups, mbarriers. Used by the
// weight-gradient GEMMs of the MLP backward (network.cu: k_ngp_bwd3).
//
// Operand layout (both operands are "MN-major": for every staged sample row k the M (or N) channel values are contiguous),
// no swizzle. In units of 16 bytes (T = 8 halves) the canonical layout the hardware expects is
//     ((8, m), (8, k)) : ((1 elem, SBO), (16 B, LBO))
// i.e. 8 channels x 8 rows form a 128-byte core matrix (row r of it at +16 r bytes, channel c at +2 c bytes); core matrices
// that are neighbours along the channels are SBO bytes apart, neighbours along the rows LBO bytes apart. A [rows][C]
// activation tile is stored with SBO = 128 B and LBO = C/8 * 128 B:
//     offset(row, ch) = (row / 8) * LBO + (ch / 8) * 128 + (row % 8) * 16 + (ch % 8) * 2      [bytes]
// One wgmma m64nNk16 consumes K = 16 rows (two core matrices along K); advancing K by 16 = start address + 2 LBO.
// Descriptor and canonical layouts: PTX ISA, warpgroup-level MMA section. Accumulator layout (m64nN, f32): thread t holds rows
// 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 j + 2 (t % 4) (+ 1): d[4 j + {0, 1}] row r, d[4 j + {2, 3}] row r + 8.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

__device__ __forceinline__ uint64_t wgmma_smem_desc(const void* smem, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem);
    uint64_t d = 0;
    d |= (uint64_t)((a >> 4) & 0x3fffu);              // start address, bits [0,14)
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;  // leading byte offset, bits [16,30)
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32;  // stride byte offset, bits [32,46)
    return d;                                           // base offset 0, layout type 0 = no swizzle (bits [62,64))
}

// D[64][N] += A^T B for one K = 16 step: A, B fp16 MN-major (transposed) operands in shared memory, D fp32 in registers.
// Every thread of the warpgroup executes it with its own fragment of D.
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc);
template <>
__device__ __forceinline__ void wgmma_f16<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(1)
        : "memory");
}
template <>
__device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(1)
        : "memory");
}
template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(1)
        : "memory");
}

// order this thread's register accesses before the wgmma that follows (required before the first wgmma of a batch)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups of this thread are still pending
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the compiler from moving accesses of an accumulator register across the asynchronous MMA
template <int R>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (the tensor core reads the operands through it)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t* mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(mbar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* mbar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((uint32_t)__cvta_generic_to_shared(mbar)) : "memory");
}
// spin until the phase with the given parity has completed; traps after ~2 s (a lost arrival must fail the launch
// loudly, not hang the GPU)
__device__ __forceinline__ void mbar_wait(uint64_t* mbar, uint32_t parity) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(mbar);
    const long long t0 = clock64();
    for (;;) {
        uint32_t done;
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n"
            : "=r"(done)
            : "r"(a), "r"(parity)
            : "memory");
        if (done) return;
        if (clock64() - t0 > 4000000000ll) asm volatile("trap;");
    }
}
