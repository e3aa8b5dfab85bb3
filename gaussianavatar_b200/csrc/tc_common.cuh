// Hopper (sm_90a) tensor-core plumbing written directly in PTX: cp.async staging and the warp-level TF32 MMA
// (mma.sync m16n8k8, fp32 accumulators in registers), with fragment loads out of the 128-byte-swizzled shared-memory images.
//
// Why mma.sync and not wgmma: TF32 wgmma reads both shared-memory operands K-major only (the transpose bits exist for 16-bit types
// alone), while the backward layer and the convolution weight gradient consume pixel-major images as they lie.  mma.sync takes its
// fragments from registers, so every image is read in whichever layout the producers wrote it.  The decoder layers move ~1 KiB per
// pixel against ~33 kFLOP (HBM bound on H100: 3.35 TB/s x 33 FLOP/B is a fraction of the TF32 rate), so the instruction's peak is
// not the limit.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace ga {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 16-byte asynchronous global -> shared copy (L2 only); !valid: the 16 bytes are zero-filled and nothing is read
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16u : 0u) : "memory");
}
__device__ __forceinline__ void cp_async16_full(uint32_t dst, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// fp32 -> tf32 with round-to-nearest: add half an ulp of the 10-bit mantissa; the tensor core drops the low 13 bits itself when it
// reads the operand, so one integer add per element is all that is needed.
__device__ __forceinline__ float to_tf32(float x) { return __uint_as_float(__float_as_uint(x) + 0x1000u); }
__device__ __forceinline__ float4 to_tf32(float4 v) { return make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w)); }

// D[16x8] += A[16x8] * B[8x8], TF32 in, fp32 accumulate.  With g = lane / 4, t = lane % 4:
//   a = {A(g, t), A(g+8, t), A(g, t+4), A(g+8, t+4)},  b = {B(t, g), B(t+4, g)},  d = {D(g, 2t), D(g, 2t+1), D(g+8, 2t), D(g+8, 2t+1)}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t lds32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// ---- image layouts -----------------------------------------------------------------------------------------------------
// K-major image: rows of 128 B (32 fp32 of K) with the 128-byte swizzle (16-byte unit XOR row % 8); a 32-wide K chunk of `rows`
// rows is one block, the next chunk follows `chunk_bytes` further.
__device__ __forceinline__ uint32_t sw128_offset(int r, int u) { return (uint32_t)r * 128u + (uint32_t)((u ^ (r & 7)) << 4); }
__device__ __forceinline__ uint32_t kmajor_off(int r, int k, uint32_t chunk_bytes)
{
    return (uint32_t)(k >> 5) * chunk_bytes + sw128_offset(r, (k & 31) >> 2) + (uint32_t)(k & 3) * 4u;
}
// Pixel-major ("MN-major") image: one 128-byte row per K index (pixel) holding 32 fp32 of M/N, the 32-byte pieces XOR row % 4;
// the next 32 M/N elements follow `chunk_bytes` further.
__device__ __forceinline__ uint32_t mn_unit(int r, int v) { return (uint32_t)r * 128u + (uint32_t)((((v >> 1) ^ (r & 3)) << 5) | ((v & 1) << 4)); }
__device__ __forceinline__ uint32_t mnmajor_off(int k, int mn, uint32_t chunk_bytes)
{
    return (uint32_t)(mn >> 5) * chunk_bytes + (uint32_t)k * 128u + (uint32_t)(((((mn & 31) >> 3) ^ (k & 3)) << 5) + (mn & 7) * 4);
}

}  // namespace tc
}  // namespace ga
