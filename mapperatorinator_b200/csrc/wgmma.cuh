// Hopper warpgroup MMA (wgmma.mma_async, kind tf32) primitives shared by the tensor-core GEMM (gemm_tc.cu) and the tensor-core
// flash attention (attention_tc.cu).  Operands in shared memory are K-major tiles of 32 fp32 per 128-byte row, written by TMA with
// SWIZZLE_128B (8-row / 1024-byte swizzle atoms); a k8 step inside an atom is a 32-byte advance of the descriptor start address.
//
// Register fragments of one warpgroup (warp w = 0..3 of the group, lane = 4 * gid + tig):
//   accumulator m64nN : d[4j + 0..3] = (16w + gid, 8j + 2tig), (16w + gid, 8j + 2tig + 1), (16w + gid + 8, 8j + 2tig), (16w + gid + 8, 8j + 2tig + 1)
//   A operand  m64k8  : a[0..3]      = (16w + gid, tig), (16w + gid + 8, tig), (16w + gid, tig + 4), (16w + gid + 8, tig + 4)
#pragma once
#include <cuda_runtime.h>

namespace mb200 {

// K-major SWIZZLE_128B shared-memory matrix descriptor: start >> 4 | LBO (unused when swizzled) | SBO = 1024 B >> 4 | layout SW128
__device__ __forceinline__ unsigned long long gmma_desc(unsigned smem_addr) {
    unsigned long long d = 0;
    d |= (unsigned long long)((smem_addr & 0x3FFFF) >> 4);
    d |= (unsigned long long)1 << 16;
    d |= (unsigned long long)(1024 >> 4) << 32;
    d |= (unsigned long long)1 << 62;
    return d;
}

__device__ __forceinline__ void gmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void gmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void gmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMA's issue / wait
template <int R>
__device__ __forceinline__ void gmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D(64x128) (+)= A(64x8, smem) . B(128x8, smem)^T
__device__ __forceinline__ void gmma_m64n128k8_ss(float (&d)[64], unsigned long long da, unsigned long long db, unsigned scale_d) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %66, 0; wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, "
        "%9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, "
        "%35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, "
        "%61, %62, %63}, %64, %65, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}

// D(64x64) (+)= A(64x8, smem) . B(64x8, smem)^T
__device__ __forceinline__ void gmma_m64n64k8_ss(float (&d)[32], unsigned long long da, unsigned long long db, unsigned scale_d) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %34, 0; wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, "
        "%9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}

// D(64x64) (+)= A(64x8, registers: tf32 bit patterns in the A-fragment layout above) . B(64x8, smem)^T
__device__ __forceinline__ void gmma_m64n64k8_rs(float (&d)[32], const unsigned (&a)[4], unsigned long long db, unsigned scale_d) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %37, 0; wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, "
        "%9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

}  // namespace mb200
