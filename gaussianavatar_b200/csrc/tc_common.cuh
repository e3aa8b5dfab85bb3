// Hopper (sm_90a) tensor-core plumbing written directly in PTX: cp.async staging, the 128-byte-swizzled shared-memory images and
// their address helpers, and two ways of multiplying them:
//   * wgmma.mma_async (TF32 in, fp32 accumulate, one warpgroup per m64 slab), used by the decoder-MLP layers (mlp_tc.cu): A in
//     registers, B read by the tensor cores through a shared-memory matrix descriptor.  TF32 wgmma reads shared-memory operands
//     K-major only, so every image a descriptor points at is K-major (the backward layer writes its X tile transposed for that);
//     the mbarrier / setmaxnreg wrappers serve the warp-specialised pipeline around it, and the TMA wrappers (tensor store,
//     reduce-add and load of a 128-byte-swizzled box, bulk-group waits) move the layers' output tiles, which are staged in the
//     same K-major layout.
//   * mma.sync m16n8k8 with fragments from ld.shared, kept only by the convolutions (conv_tc.cu): their weight gradient reads the
//     pixel-major images as they lie, which TF32 wgmma cannot.
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

// ---- wgmma (warpgroup MMA) ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major operand in the 128-byte-swizzled layout above (rows of 128 B = 32 TF32 along K,
// 8-row atoms of 1024 B): start address >> 4 (bits 0-13), leading byte offset 1 (unused by swizzled K-major layouts: one k-step
// never leaves the 128-byte row), stride byte offset 1024 >> 4 (bits 32-45: the next 8 rows of M/N), base offset 0, swizzle mode
// 1 = 128 B (bits 62-63).  The hardware applies the swizzle to address bits 4-6 from bits 7-9, so images start on 1024-byte
// boundaries and a k-step inside the atom simply advances the start address (kstep_addr).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr)
{
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024u >> 4) << 32) | ((uint64_t)1 << 62);
}
// start address of k-step ks (8 TF32 = 32 bytes of K) of a K-major image whose 32-wide K chunks lie chunk_bytes apart
__device__ __forceinline__ uint32_t kstep_addr(uint32_t base, int ks, uint32_t chunk_bytes)
{
    return base + (uint32_t)(ks >> 2) * chunk_bytes + (uint32_t)(ks & 3) * 32u;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving a register read by / written by an in-flight wgmma across the wait that retires it
template <int R, int C> __device__ __forceinline__ void wgmma_fence_operand(float (&d)[R][C])
{
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
        for (int j = 0; j < C; ++j) asm volatile("" : "+f"(d[i][j])::"memory");
}
template <int R, int C> __device__ __forceinline__ void wgmma_fence_operand(uint32_t (&d)[R][C])
{
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
        for (int j = 0; j < C; ++j) asm volatile("" : "+r"(d[i][j])::"memory");
}

// D[64 x N] += A[64 x 8] * B[8 x N] for one warpgroup, TF32 in, fp32 accumulate.  A comes from registers: warp w % 4 of the group
// holds rows 16 (w % 4) .. + 15 as the m16n8k8 A fragment (mma_tf32 above).  B is read through a descriptor (wgmma_desc).  d[nt]
// is the m16n8k8 accumulator fragment of columns 8 nt .. 8 nt + 7 of the warp's 16 rows.
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[4][4], const uint32_t (&a)[4], uint64_t b)
{
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
                 : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]),
                   "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]),
                   "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]),
                   "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[8][4], const uint32_t (&a)[4], uint64_t b)
{
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}\n"
                 : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]),
                   "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]),
                   "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]),
                   "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]),
                   "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]),
                   "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]),
                   "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]),
                   "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[16][4], const uint32_t (&a)[4], uint64_t b)
{
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}\n"
                 : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]),
                   "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]),
                   "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]),
                   "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]),
                   "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]),
                   "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]),
                   "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]),
                   "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3]),
                   "+f"(d[8][0]), "+f"(d[8][1]), "+f"(d[8][2]), "+f"(d[8][3]),
                   "+f"(d[9][0]), "+f"(d[9][1]), "+f"(d[9][2]), "+f"(d[9][3]),
                   "+f"(d[10][0]), "+f"(d[10][1]), "+f"(d[10][2]), "+f"(d[10][3]),
                   "+f"(d[11][0]), "+f"(d[11][1]), "+f"(d[11][2]), "+f"(d[11][3]),
                   "+f"(d[12][0]), "+f"(d[12][1]), "+f"(d[12][2]), "+f"(d[12][3]),
                   "+f"(d[13][0]), "+f"(d[13][1]), "+f"(d[13][2]), "+f"(d[13][3]),
                   "+f"(d[14][0]), "+f"(d[14][1]), "+f"(d[14][2]), "+f"(d[14][3]),
                   "+f"(d[15][0]), "+f"(d[15][1]), "+f"(d[15][2]), "+f"(d[15][3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}

// ---- mbarrier / warpgroup register split -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// waits for the completion of the barrier phase with this parity (phase k of a barrier has parity k & 1)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
// arms the barrier's current phase for `bytes` of asynchronous copies (one arrival)
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// generic-proxy shared-memory writes (st.shared) made visible to the async proxy (wgmma operand reads, TMA stores)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- TMA (bulk tensor copies) ------------------------------------------------------------------------------------------
// `tmap` is the address of a CUtensorMap kernel parameter (__grid_constant__) of a 2-D fp32 matrix with 128-byte-swizzled boxes of
// 32 columns x `rows` rows; coordinates are {column, row}.  In shared memory such a box is one chunk of the K-major image above:
// element (row r, column k) at sw128_offset(r, k / 4) + (k % 4) * 4, the box starting on a 1024-byte boundary.  Rows and columns
// outside the matrix are not written by a store and read as zeros by a load.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void *tmap, uint32_t bar, int col, int row)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tmap), "r"(bar), "r"(col), "r"(row) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void *tmap, uint32_t src, int col, int row)
{
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tmap), "r"(src), "r"(col), "r"(row)
                 : "memory");
}
// global += box, added in L2 (f32: round to nearest even, subnormal inputs and results flushed to sign-preserving zero)
__device__ __forceinline__ void tma_reduce_add_2d(const void *tmap, uint32_t src, int col, int row)
{
    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tmap), "r"(src), "r"(col),
                 "r"(row) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still READ their shared-memory source (the buffer may be rewritten)
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// at most N of this thread's bulk groups are incomplete (their global writes not yet performed)
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// barrier of the 128 threads of one warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

}  // namespace tc
}  // namespace ga
