// Warp-level tensor-core MMA (mma.sync), shared by the interaction kernels, the GRU recurrence kernels and the self-attention kernels.
// Hardware only: the emulation build compiles the SIMT kernels and leaves these out.
#pragma once
#ifndef DR_CUDA_EMU
#include <stdint.h>

namespace drc {

// c[16 x 8] += a[16 x 16] b[16 x 8], bf16 operands, fp32 accumulators (row.col fragment layout of the PTX ISA)
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// c[16 x 8] += a[16 x 8] b[8 x 8]: the first k8 half of the m16n8k16 fragments (a0 rows g, a1 rows g + 8; b0 k rows 2t, 2t + 1)
__device__ __forceinline__ void mma_bf16_1688(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(b0));
}

}  // namespace drc
#endif
