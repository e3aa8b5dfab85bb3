// LPIPS (lpips.LPIPS(net='alex', version='0.1'), eval mode) forward and input gradient on sm_90a.
//
// Network (torchvision alexnet().features sliced as lpips does; every map NHWC fp32, rendered and ground-truth images in one launch):
//   conv1 11x11/4 pad 2 (3->64) relu | pool 3/2 | conv2 5x5 pad 2 (64->192) relu | pool 3/2 | conv3 3x3 (192->384) relu |
//   conv4 3x3 (384->256) relu | conv5 3x3 (256->256) relu
// and per relu map k:  d_k = mean_px sum_c w_k,c (f0_c / (|f0| + 1e-10) - f1_c / (|f1| + 1e-10))^2,  out = sum_k d_k.
//
// Every convolution is one implicit GEMM on wgmma TF32 (fp32 accumulate): rows = output pixels of all images (128 per CTA), columns =
// output channels (BN per CTA), K = taps x input channels, both operands K-major 128-byte-swizzled shared-memory images (tc_common.cuh).
// A producer warpgroup gathers the im2col rows with cp.async (a 32-wide K chunk of an NHWC map is one tap's 32 contiguous channels; a
// tap outside the map is zero-filled) and the weight rows, rounds the weights to TF32 in place, and hands each stage to two consumer
// warpgroups (64 rows each) through mbarriers.  conv1's producer gathers the 11x11x3 window from the planar images instead and applies
// the input affine (scaling layer composed with the caller's in_scale / in_shift) while it does; the padding is zero after the affine.
// The data gradients of conv5..conv2 are the same kernel over dZ with the flipped, transposed weights (stride 1, 'same' padding).
//
// Nothing here uses atomics: every output element has one fixed summation order, so values and gradients are bit-reproducible, and a
// frame's result does not depend on the other frames of the batch.
#include <utility>

#include "common.cuh"
#include "tc_common.cuh"

namespace ga {
namespace {

using namespace tc;

constexpr size_t kMaxSmem = 232448;
constexpr int kThreads = 384;          // producer warpgroup + two consumer warpgroups
constexpr int kBM = 128;               // output pixels per CTA
constexpr int kStages = 6, kLook = 4;  // K chunks of 32 in flight
static_assert(kLook <= kStages - 2, "lookahead must leave the stages being converted and read alone");
constexpr int kAChunk = kBM * 128;     // 16 KB: [128 rows][32 fp32]
constexpr int kDistWarps = 8;
constexpr int kMaxPart = 128;          // per-image partial sums of a distance launch
constexpr float kEps = 1e-10f;

// lpips ScalingLayer: x = (in - shift) / scale
constexpr float kShift[3] = {-.030f, -.088f, -.188f}, kScale[3] = {.458f, .448f, .450f};
__constant__ float c_scale[3] = {kScale[0], kScale[1], kScale[2]};

// fp32 -> TF32, round to nearest (ties away), low 13 mantissa bits cleared: the stored maps are exact TF32 operands
__device__ __forceinline__ float tf32_rn(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

__device__ __forceinline__ void wgmma_ss_n64(float (&d)[8][4], uint64_t a, uint64_t b)
{
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
                 : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]),
                   "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]),
                   "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]),
                   "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]),
                   "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]),
                   "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]),
                   "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]),
                   "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3])
                 : "l"(a), "l"(b), "r"(1));
}
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[16][4], uint64_t a, uint64_t b)
{
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
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
                 : "l"(a), "l"(b), "r"(1));
}
template <int BN> __device__ __forceinline__ void wgmma_ss(float (&d)[BN / 8][4], uint64_t a, uint64_t b)
{
    if constexpr (BN == 64) wgmma_ss_n64(d, a, b);
    else wgmma_ss_n128(d, a, b);
}

// ---- implicit-GEMM convolution ------------------------------------------------------------------------------------------
struct ConvParams {
    const float *in0, *in1;   // NHWC [imgs][Hi][Wi][Cin]; planar: [imgs][3][Hi][Wi], images >= nsplit read from in1
    int nsplit, planar;
    float a[3], b[3];         // planar: per-channel input affine
    const float *W; int K;    // [N][K], k = tap * Cin + ci (planar: tap * 3 + c, zero from 363 to K)
    const float *bias;        // nullable: no bias, no ReLU, no rounding (data gradients)
    float *out; int N;        // NHWC [P][N]
    int Hi, Wi, Cin, Ho, Wo, KS, stride, pad, P;
};

template <int BN> struct alignas(1024) ConvSmem {
    unsigned char a[kStages][kAChunk];       // im2col rows, K-major
    unsigned char b[kStages][BN * 128];      // weight rows, K-major
    uint64_t full[kStages], empty[kStages];  // producer -> consumers (128 arrivals), consumers -> producer (256 arrivals)
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1) lpips_conv_kernel(const __grid_constant__ ConvParams p)
{
    extern __shared__ unsigned char smem_raw[];
    ConvSmem<BN> &sm = *reinterpret_cast<ConvSmem<BN> *>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
    const int nchunks = p.K / 32;
    if (tid < kStages) { mbar_init(smem_u32(&sm.full[tid]), 128); mbar_init(smem_u32(&sm.empty[tid]), 256); }
    fence_proxy_async();
    __syncthreads();

    if (warp < 4) {
        // ---- producer: thread owns 16-byte unit u of rows r = tid / 8 + 16 i of the A chunk (i < 8) and of the B chunk (i < BN / 16)
        const int u = tid & 7, rb = tid >> 3;
        const int HWo = p.Ho * p.Wo;
        const float *img[8];
        int iy0[8], ix0[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = m0 + rb + 16 * i;
            const bool ok = m < p.P;
            const int n = ok ? m / HWo : 0, rem = ok ? m - n * HWo : 0;
            const int oy = rem / p.Wo, ox = rem - oy * p.Wo;
            iy0[i] = ok ? oy * p.stride - p.pad : -(1 << 20);       // rows past P: every tap out of bounds (zero-filled)
            ix0[i] = ox * p.stride - p.pad;
            if (p.planar) img[i] = (n < p.nsplit ? p.in0 + (size_t)n * 3 * p.Hi * p.Wi : p.in1 + (size_t)(n - p.nsplit) * 3 * p.Hi * p.Wi);
            else img[i] = p.in0 + (size_t)n * p.Hi * p.Wi * p.Cin;
        }
        const int cpt = p.Cin / 32;                                  // K chunks per tap (NHWC)
        const uint32_t a0s = smem_u32(sm.a[0]), b0s = smem_u32(sm.b[0]);
        auto issue = [&](int j) {
            const int st = j % kStages;
            if (j < nchunks && j >= kStages) mbar_wait(smem_u32(&sm.empty[st]), ((j / kStages) & 1) ^ 1);
            if (j < nchunks) {
                const uint32_t da = a0s + (uint32_t)st * kAChunk, db = b0s + (uint32_t)st * (BN * 128);
                if (!p.planar) {
                    const int tap = j / cpt, ci = (j - tap * cpt) * 32 + 4 * u;
                    const int ky = tap / p.KS, kx = tap - ky * p.KS;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int iy = iy0[i] + ky, ix = ix0[i] + kx;
                        const bool ok = iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi;
                        const float *src = ok ? img[i] + ((size_t)iy * p.Wi + ix) * p.Cin + ci : p.in0;
                        cp_async16(da + sw128_offset(rb + 16 * i, u), src, ok);
                    }
                } else {
                    // conv1: element k = tap * 3 + c of the 11x11x3 window, affine applied here, zero outside the image and past K = 363
                    int off[4], kyv[4], kxv[4];
                    float av[4], bv[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int k = j * 32 + 4 * u + e;
                        const int tap = k / 3, c = k - tap * 3;
                        const bool kin = k < 363;
                        kyv[e] = kin ? tap / 11 : (1 << 20);
                        kxv[e] = tap % 11;
                        off[e] = c * p.Hi * p.Wi;
                        av[e] = p.a[c < 3 ? c : 0]; bv[e] = p.b[c < 3 ? c : 0];
                    }
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        float v[4];
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int iy = iy0[i] + kyv[e], ix = ix0[i] + kxv[e];
                            const bool ok = iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi;
                            v[e] = ok ? tf32_rn(fmaf(av[e], __ldg(img[i] + off[e] + (size_t)iy * p.Wi + ix), bv[e])) : 0.f;
                        }
                        *reinterpret_cast<float4 *>(sm.a[st] + sw128_offset(rb + 16 * i, u)) = make_float4(v[0], v[1], v[2], v[3]);
                    }
                }
                const float *wsrc = p.W + (size_t)(n0 + rb) * p.K + j * 32 + 4 * u;
#pragma unroll
                for (int i = 0; i < BN / 16; ++i) cp_async16_full(db + sw128_offset(rb + 16 * i, u), wsrc + (size_t)16 * i * p.K);
            }
            cp_async_commit();                                      // one group per chunk (empty past the end): uniform wait counts
        };
        for (int j = 0; j < kLook; ++j) issue(j);
        for (int j = 0; j < nchunks; ++j) {
            const int st = j % kStages;
            cp_async_wait<kLook - 1>();
#pragma unroll
            for (int i = 0; i < BN / 16; ++i) {                      // weights to TF32, in place (each thread its own copies)
                float4 *w = reinterpret_cast<float4 *>(sm.b[st] + sw128_offset(rb + 16 * i, u));
                float4 x = *w;
                *w = make_float4(tf32_rn(x.x), tf32_rn(x.y), tf32_rn(x.z), tf32_rn(x.w));
            }
            fence_proxy_async();                                    // generic-proxy writes and landed copies -> tensor-core reads
            mbar_arrive(smem_u32(&sm.full[st]));
            issue(j + kLook);
        }
        cp_async_wait<0>();
        return;
    }

    // ---- consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63
    const int wg = (warp >> 2) - 1, g = lane >> 2, t4 = lane & 3;
    float acc[BN / 8][4];
#pragma unroll
    for (int nt = 0; nt < BN / 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
    const uint32_t a0s = smem_u32(sm.a[0]) + (uint32_t)wg * (64 * 128), b0s = smem_u32(sm.b[0]);
    for (int j = 0; j < nchunks; ++j) {
        const int st = j % kStages;
        mbar_wait(smem_u32(&sm.full[st]), (j / kStages) & 1);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
            wgmma_ss<BN>(acc, wgmma_desc(a0s + (uint32_t)st * kAChunk + 32u * ks), wgmma_desc(b0s + (uint32_t)st * (BN * 128) + 32u * ks));
        wgmma_commit();
        wgmma_wait<1>();                                            // chunk j - 1 retired: its stage goes back to the producer
        if (j > 0) mbar_arrive(smem_u32(&sm.empty[(j - 1) % kStages]));
    }
    wgmma_wait<0>();
    wgmma_fence_operand(acc);

    // acc[nt] = {Y(r, c), Y(r, c + 1), Y(r + 8, c), Y(r + 8, c + 1)}, r = 64 wg + 16 (warp % 4) + g, c = 8 nt + 2 t4
    const int r = m0 + 64 * wg + 16 * (warp & 3) + g;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = r + 8 * h;
        if (m >= p.P) continue;
        float *o = p.out + (size_t)m * p.N + n0;
#pragma unroll
        for (int nt = 0; nt < BN / 8; ++nt) {
            const int c = 8 * nt + 2 * t4;
            float v0 = acc[nt][2 * h], v1 = acc[nt][2 * h + 1];
            if (p.bias) {
                v0 = tf32_rn(fmaxf(v0 + __ldg(p.bias + n0 + c), 0.f));
                v1 = tf32_rn(fmaxf(v1 + __ldg(p.bias + n0 + c + 1), 0.f));
            }
            *reinterpret_cast<float2 *>(o + c) = make_float2(v0, v1);
        }
    }
}

// ---- max pool 3/2 (NHWC): first maximum in row-major window order, as torch.max_pool2d ------------------------------------
__global__ void lpips_pool_kernel(const float *__restrict__ in, float *__restrict__ out, uint8_t *__restrict__ arg, int imgs, int Hi, int Wi,
                                  int C, int Ho, int Wo)
{
    const long long total = (long long)imgs * Ho * Wo * C;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(e % C);
        const long long q = e / C;
        const int ox = (int)(q % Wo), oy = (int)((q / Wo) % Ho), n = (int)(q / ((long long)Wo * Ho));
        const float *src = in + (((size_t)n * Hi + 2 * oy) * Wi + 2 * ox) * C + c;
        float best = src[0];
        int bi = 0;
#pragma unroll
        for (int t = 1; t < 9; ++t) {
            const float v = src[((size_t)(t / 3) * Wi + t % 3) * C];
            if (v > best || isnan(v)) { best = v; bi = t; }
            if (isnan(best)) break;
        }
        out[e] = best;
        arg[e] = (uint8_t)bi;
    }
}

// backward: each input element gathers the (<= 4) windows that chose it, in window order
__global__ void lpips_unpool_kernel(const float *__restrict__ gout, const uint8_t *__restrict__ arg, float *__restrict__ gin, int imgs, int Hi,
                                    int Wi, int C, int Ho, int Wo)
{
    const long long total = (long long)imgs * Hi * Wi * C;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(e % C);
        const long long q = e / C;
        const int ix = (int)(q % Wi), iy = (int)((q / Wi) % Hi), n = (int)(q / ((long long)Wi * Hi));
        const int oy0 = max(0, (iy - 1) / 2), oy1 = min(Ho - 1, iy / 2), ox0 = max(0, (ix - 1) / 2), ox1 = min(Wo - 1, ix / 2);
        float s = 0.f;
        for (int oy = oy0; oy <= oy1; ++oy)
            for (int ox = ox0; ox <= ox1; ++ox) {
                const size_t o = (((size_t)n * Ho + oy) * Wo + ox) * C + c;
                if (arg[o] == (iy - 2 * oy) * 3 + (ix - 2 * ox)) s += gout[o];
            }
        gin[e] = s;
    }
}

// ---- distance of one layer: per pixel, warp over channels; per-CTA partial sums (deterministic order) ----------------------
template <int J>
__global__ void __launch_bounds__(32 * kDistWarps) lpips_dist_kernel(const float *__restrict__ f, const float *__restrict__ lin, int B, int HW,
                                                                  float *__restrict__ part)
{
    __shared__ float red[kDistWarps];
    constexpr int C = 32 * J;
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float w[J];
#pragma unroll
    for (int j = 0; j < J; ++j) w[j] = __ldg(lin + lane + 32 * j);
    const float *f0 = f + (size_t)b * HW * C, *f1 = f + (size_t)(B + b) * HW * C;
    float acc = 0.f;
    for (int px = blockIdx.x * kDistWarps + warp; px < HW; px += gridDim.x * kDistWarps) {
        float x0[J], x1[J], s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            x0[j] = f0[(size_t)px * C + lane + 32 * j]; x1[j] = f1[(size_t)px * C + lane + 32 * j];
            s0 = fmaf(x0[j], x0[j], s0); s1 = fmaf(x1[j], x1[j], s1);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
        const float d0 = sqrtf(s0) + kEps, d1 = sqrtf(s1) + kEps;
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < J; ++j) { const float h = x0[j] / d0 - x1[j] / d1; d = fmaf(w[j] * h, h, d); }
#pragma unroll
        for (int o = 16; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        acc += d;
    }
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < kDistWarps; ++i) s += red[i];
        part[b * kMaxPart + blockIdx.x] = s;
    }
}

struct SumParams {
    const float *part[5];
    int nblk[5], HW[5];
    int B;
    float *out;
    float *in_scale_ws, in_scale;
};

// out[b] = sum_k (sum of layer k's partials, in CTA order) / HW_k; also records the input scale for the backward
__global__ void lpips_sum_kernel(const __grid_constant__ SumParams p)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0) *p.in_scale_ws = p.in_scale;
    if (b >= p.B) return;
    float v = 0.f;
    for (int k = 0; k < 5; ++k) {
        float s = 0.f;
        for (int i = 0; i < p.nblk[k]; ++i) s += p.part[k][b * kMaxPart + i];
        v += s / (float)p.HW[k];
    }
    p.out[b] = v;
}

// ---- backward of one layer's distance term through the normalisation, plus the next slice's gradient, times the ReLU mask -----
// dZ = [f0 > 0] (gnext + gd),  gd_c = gh_c / d0 - f0_c (sum_j gh_j f0_j) / (n0 d0^2)  (0 where n0 = 0),
// gh_c = 2 (g[b] / HW) w_c (f0_c / d0 - f1_c / d1)
template <int J>
__global__ void __launch_bounds__(32 * kDistWarps) lpips_dnorm_kernel(const float *__restrict__ f, const float *__restrict__ lin,
                                                                   const float *__restrict__ g, const float *__restrict__ gnext, int B, int HW,
                                                                   float *__restrict__ dz)
{
    constexpr int C = 32 * J;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long q = (long long)blockIdx.x * kDistWarps + warp;
    if (q >= (long long)B * HW) return;
    const int b = (int)(q / HW), px = (int)(q - (long long)b * HW);
    const float *f0 = f + ((size_t)b * HW + px) * C, *f1 = f + ((size_t)(B + b) * HW + px) * C;
    const float sc = 2.f * __ldg(g + b) / (float)HW;
    float x0[J], x1[J], s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
        x0[j] = f0[lane + 32 * j]; x1[j] = f1[lane + 32 * j];
        s0 = fmaf(x0[j], x0[j], s0); s1 = fmaf(x1[j], x1[j], s1);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
    const float n0 = sqrtf(s0), d0 = n0 + kEps, d1 = sqrtf(s1) + kEps;
    float gh[J], dot = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
        gh[j] = sc * __ldg(lin + lane + 32 * j) * (x0[j] / d0 - x1[j] / d1);
        dot = fmaf(gh[j], x0[j], dot);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    const float k2 = n0 > 0.f ? dot / (n0 * d0 * d0) : 0.f;
    float *o = dz + ((size_t)b * HW + px) * C;
    const float *gn = gnext ? gnext + ((size_t)b * HW + px) * C : nullptr;
#pragma unroll
    for (int j = 0; j < J; ++j) {
        float v = n0 > 0.f ? gh[j] / d0 - x0[j] * k2 : 0.f;
        if (gn) v += gn[lane + 32 * j];
        o[lane + 32 * j] = x0[j] > 0.f ? tf32_rn(v) : 0.f;
    }
}

// ---- conv1 image gradient on the CUDA cores: one thread per input pixel of one stride phase (the <= 3 x 3 taps that reach it
// are the same for the whole CTA, so their weights sit in shared memory and every read is a broadcast) --------------------------
constexpr int kImgThreads = 128;
__global__ void __launch_bounds__(kImgThreads) lpips_img_grad_kernel(const float *__restrict__ dz1, const float *__restrict__ w1,
                                                                  const float *__restrict__ in_scale, int H, int W, int H1, int W1,
                                                                  float *__restrict__ d_in)
{
    __shared__ float ws[9][64][3];
    const int ph = blockIdx.y, ry = ph >> 2, rx = ph & 3, b = blockIdx.z;
    const int qy = (ry + 2) & 3, qx = (rx + 2) & 3;           // first tap of the phase: (y + 2 - ky) % 4 == 0
    const int nky = qy + 8 <= 10 ? 3 : 2, nkx = qx + 8 <= 10 ? 3 : 2;
    for (int i = threadIdx.x; i < nky * nkx * 64 * 3; i += kImgThreads) {
        const int c = i % 3, oc = (i / 3) % 64, t = i / 192;
        const int ky = qy + 4 * (t / nkx), kx = qx + 4 * (t % nkx);
        ws[t][oc][c] = __ldg(w1 + (size_t)oc * 384 + (ky * 11 + kx) * 3 + c);
    }
    __syncthreads();
    const int Wq = (W + 3) / 4;
    const int idx = blockIdx.x * kImgThreads + threadIdx.x;
    const int y = 4 * (idx / Wq) + ry, x = 4 * (idx % Wq) + rx;
    if (y >= H || x >= W) return;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int ty = 0; ty < nky; ++ty) {
        const int oy = (y + 2 - qy - 4 * ty) / 4;                // exact: y + 2 - ky is a multiple of 4
        if (y + 2 - qy - 4 * ty < 0 || oy >= H1) continue;
        for (int tx = 0; tx < nkx; ++tx) {
            const int ox = (x + 2 - qx - 4 * tx) / 4;
            if (x + 2 - qx - 4 * tx < 0 || ox >= W1) continue;
            const float4 *z = reinterpret_cast<const float4 *>(dz1 + (((size_t)b * H1 + oy) * W1 + ox) * 64);
            const float(*wt)[3] = ws[ty * nkx + tx];
#pragma unroll 4
            for (int o4 = 0; o4 < 16; ++o4) {
                const float4 v = __ldg(z + o4);
                const float zz[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    a0 = fmaf(zz[e], wt[4 * o4 + e][0], a0);
                    a1 = fmaf(zz[e], wt[4 * o4 + e][1], a1);
                    a2 = fmaf(zz[e], wt[4 * o4 + e][2], a2);
                }
            }
        }
    }
    const float s = *in_scale;
    const size_t plane = (size_t)H * W, o = (size_t)b * 3 * plane + (size_t)y * W + x;
    d_in[o] = a0 * (s / c_scale[0]);
    d_in[o + plane] = a1 * (s / c_scale[1]);
    d_in[o + 2 * plane] = a2 * (s / c_scale[2]);
}

// ---- geometry, weights and workspace ---------------------------------------------------------------------------------------
constexpr int kCin[5] = {3, 64, 192, 384, 256}, kCout[5] = {64, 192, 384, 256, 256}, kKS[5] = {11, 5, 3, 3, 3};
constexpr int kK1 = 384;               // conv1's K = 363 padded to whole 32-wide chunks with zero weights

struct WeightLayout {
    size_t w[5], b[5], wd[5], lin[5], total;   // wd[0] unused: conv1's image gradient reads w[0]
    WeightLayout()
    {
        size_t o = 0;
        for (int l = 0; l < 5; ++l) {
            w[l] = o; o += (size_t)kCout[l] * (l == 0 ? kK1 : kKS[l] * kKS[l] * kCin[l]);
            b[l] = o; o += kCout[l];
        }
        wd[0] = 0;
        for (int l = 1; l < 5; ++l) { wd[l] = o; o += (size_t)kCout[l] * kKS[l] * kKS[l] * kCin[l]; }
        for (int l = 0; l < 5; ++l) { lin[l] = o; o += kCout[l]; }
        total = o;
    }
};

struct Geo {
    int B, H, W;
    int h[5], w[5];          // relu map k
    int ph[2], pw[2];        // pool k output
    Geo(int B_, int H_, int W_) : B(B_), H(H_), W(W_)
    {
        h[0] = (H + 4 - 11) / 4 + 1; w[0] = (W + 4 - 11) / 4 + 1;
        ph[0] = (h[0] - 3) / 2 + 1; pw[0] = (w[0] - 3) / 2 + 1;
        h[1] = ph[0]; w[1] = pw[0];
        ph[1] = (h[1] - 3) / 2 + 1; pw[1] = (w[1] - 3) / 2 + 1;
        h[2] = h[3] = h[4] = ph[1]; w[2] = w[3] = w[4] = pw[1];
    }
    size_t map(int k, int imgs) const { return (size_t)imgs * h[k] * w[k] * kCout[k]; }
    size_t pool(int k, int imgs) const { return (size_t)imgs * ph[k] * pw[k] * kCout[k]; }
    int nblk(int k) const { const int n = cdiv((long long)h[k] * w[k], 64); return n < kMaxPart ? n : kMaxPart; }
};

// the workspace regions (GaLpipsViews) carved from `ws`; returns the bytes they take (ws == nullptr: size query only)
size_t carve(const Geo &g, void *ws, GaLpipsViews *v)
{
    Carver c(ws);
    const int B2 = 2 * g.B;
    for (int k = 0; k < 5; ++k) v->relu[k] = c.take<float>(g.map(k, B2));
    for (int k = 0; k < 2; ++k) { v->pool[k] = c.take<float>(g.pool(k, B2)); v->pool_arg[k] = c.take<uint8_t>(g.pool(k, B2)); }
    v->partials = c.take<float>((size_t)5 * g.B * kMaxPart);
    v->in_scale = c.take<float>(1);
    for (int k = 0; k < 5; ++k) v->dz[k] = c.take<float>(g.map(k, g.B));
    for (int k = 0; k < 4; ++k) v->dnext[k] = c.take<float>(g.map(k, g.B));
    for (int k = 0; k < 2; ++k) v->dpool[k] = c.take<float>(g.pool(k, g.B));
    return c.used();
}

const char *const kConvName[5] = {"lpips_conv1", "lpips_conv2", "lpips_conv3", "lpips_conv4", "lpips_conv5"};
const char *const kDgradName[5] = {"", "lpips_dgrad2", "lpips_dgrad3", "lpips_dgrad4", "lpips_dgrad5"};
const char *const kDistName[5] = {"lpips_dist1", "lpips_dist2", "lpips_dist3", "lpips_dist4", "lpips_dist5"};
const char *const kDnormName[5] = {"lpips_dnorm1", "lpips_dnorm2", "lpips_dnorm3", "lpips_dnorm4", "lpips_dnorm5"};
const char *const kPoolName[2] = {"lpips_pool1", "lpips_pool2"};
const char *const kUnpoolName[2] = {"lpips_unpool1", "lpips_unpool2"};

template <int BN> int launch_conv(const ConvParams &p, const char *name, cudaStream_t st)
{
    static PerDeviceOnce attr;
    constexpr int smem = (int)sizeof(ConvSmem<BN>) + 1024;
    static_assert(sizeof(ConvSmem<BN>) + 1024 <= kMaxSmem, "conv shared memory");
    if (attr.first()) GA_CHECK_CUDA(cudaFuncSetAttribute(lpips_conv_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const dim3 grid(cdiv(p.P, kBM), p.N / BN);
    {
        ProfScope _ps(name, st);
        lpips_conv_kernel<BN><<<grid, kThreads, smem, st>>>(p);
    }
    GA_CHECK_LAUNCH(name);
    return GA_OK;
}
// N = 64 or 192 (a multiple of 64 but not of 128): 64-wide column tiles; 256 and 384: 128-wide
int conv(const ConvParams &p, const char *name, cudaStream_t st)
{
    return p.N % 128 == 0 ? launch_conv<128>(p, name, st) : launch_conv<64>(p, name, st);
}

ConvParams conv_params(const float *in, int imgs, int Hi, int Wi, int l, const float *W, const float *bias, float *out, int Ho, int Wo, bool dgrad)
{
    ConvParams p{};
    p.in0 = p.in1 = in; p.nsplit = imgs; p.planar = 0;
    p.W = W; p.bias = bias; p.out = out;
    p.Cin = dgrad ? kCout[l] : kCin[l]; p.N = dgrad ? kCin[l] : kCout[l];
    p.KS = kKS[l]; p.K = p.KS * p.KS * p.Cin;
    p.stride = 1; p.pad = p.KS / 2;
    p.Hi = Hi; p.Wi = Wi; p.Ho = Ho; p.Wo = Wo; p.P = imgs * Ho * Wo;
    return p;
}

template <typename... KArgs, typename... Args>
int simple_launch(const char *name, void (*k)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args &&...args)
{
    {
        ProfScope _ps(name, st);
        k<<<grid, block, 0, st>>>(std::forward<Args>(args)...);
    }
    GA_CHECK_LAUNCH(name);
    return GA_OK;
}

int elementwise_grid(long long n) { const long long b = (n + 255) / 256; return (int)(b < 132 * 16 ? b : 132 * 16); }

int dist(int k, const Geo &g, const float *f, const float *lin, float *part, cudaStream_t st)
{
    const dim3 grid(g.nblk(k), g.B);
    const int HW = g.h[k] * g.w[k];
    switch (kCout[k] / 32) {
    case 2: return simple_launch(kDistName[k], lpips_dist_kernel<2>, grid, 32 * kDistWarps, st, f, lin, g.B, HW, part);
    case 6: return simple_launch(kDistName[k], lpips_dist_kernel<6>, grid, 32 * kDistWarps, st, f, lin, g.B, HW, part);
    case 8: return simple_launch(kDistName[k], lpips_dist_kernel<8>, grid, 32 * kDistWarps, st, f, lin, g.B, HW, part);
    default: return simple_launch(kDistName[k], lpips_dist_kernel<12>, grid, 32 * kDistWarps, st, f, lin, g.B, HW, part);
    }
}

int dnorm(int k, const Geo &g, const float *f, const float *lin, const float *gout, const float *gnext, float *dz, cudaStream_t st)
{
    const int HW = g.h[k] * g.w[k];
    const dim3 grid(cdiv((long long)g.B * HW, kDistWarps));
    switch (kCout[k] / 32) {
    case 2: return simple_launch(kDnormName[k], lpips_dnorm_kernel<2>, grid, 32 * kDistWarps, st, f, lin, gout, gnext, g.B, HW, dz);
    case 6: return simple_launch(kDnormName[k], lpips_dnorm_kernel<6>, grid, 32 * kDistWarps, st, f, lin, gout, gnext, g.B, HW, dz);
    case 8: return simple_launch(kDnormName[k], lpips_dnorm_kernel<8>, grid, 32 * kDistWarps, st, f, lin, gout, gnext, g.B, HW, dz);
    default: return simple_launch(kDnormName[k], lpips_dnorm_kernel<12>, grid, 32 * kDistWarps, st, f, lin, gout, gnext, g.B, HW, dz);
    }
}

int check_args(int B, int H, int W, const void *weights, const void *ws)
{
    GA_REQUIRE(B >= 1 && H > 0 && W > 0, "lpips: bad shape B=%d H=%d W=%d", B, H, W);
    GA_REQUIRE(H >= 31 && W >= 31, "lpips: the image must be at least 31x31 (got %dx%d): both max pools need 3 inputs", H, W);
    GA_REQUIRE((long long)B * H * W <= (1LL << 31) / 4, "lpips: B*H*W=%lld is too large", (long long)B * H * W);
    GA_REQUIRE(weights && ws, "lpips: null weights or workspace");
    GA_REQUIRE((reinterpret_cast<uintptr_t>(weights) & 15) == 0 && (reinterpret_cast<uintptr_t>(ws) & 255) == 0,
               "lpips: weights must be 16-byte and the workspace 256-byte aligned");
    return GA_OK;
}

}  // namespace
}  // namespace ga

extern "C" size_t ga_lpips_weights_floats(void) { return ga::WeightLayout().total; }

extern "C" size_t ga_lpips_workspace_bytes(int32_t B, int32_t H, int32_t W)
{
    if (B < 1 || H < 31 || W < 31) return 0;
    GaLpipsViews v;
    return ga::carve(ga::Geo(B, H, W), nullptr, &v);
}

extern "C" int ga_lpips_views(int32_t B, int32_t H, int32_t W, void *ws, GaLpipsViews *out)
{
    if (int rc = ga::check_args(B, H, W, ws, ws)) return rc;
    GA_REQUIRE(out, "lpips: null views");
    ga::carve(ga::Geo(B, H, W), ws, out);
    return GA_OK;
}

extern "C" int ga_lpips_forward(int32_t B, int32_t H, int32_t W, const float *weights, const float *in0, const float *in1, float in_scale,
                                float in_shift, void *ws, float *out, void *stream)
{
    using namespace ga;
    if (int rc = check_args(B, H, W, weights, ws)) return rc;
    GA_REQUIRE(in0 && in1 && out, "lpips: null input or output");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Geo g(B, H, W);
    const WeightLayout L;
    GaLpipsViews v;
    carve(g, ws, &v);
    const int B2 = 2 * B;
    {   // conv1 straight from the planar images, scaling layer and caller affine folded: x' = a_c x + b_c
        ConvParams p{};
        p.in0 = in0; p.in1 = in1; p.nsplit = B; p.planar = 1;
        for (int c = 0; c < 3; ++c) { p.a[c] = in_scale / kScale[c]; p.b[c] = (in_shift - kShift[c]) / kScale[c]; }
        p.W = weights + L.w[0]; p.K = kK1; p.bias = weights + L.b[0]; p.out = v.relu[0]; p.N = 64;
        p.Hi = H; p.Wi = W; p.Cin = 3; p.Ho = g.h[0]; p.Wo = g.w[0]; p.KS = 11; p.stride = 4; p.pad = 2; p.P = B2 * g.h[0] * g.w[0];
        if (int rc = conv(p, kConvName[0], st)) return rc;
    }
    const float *x = v.relu[0];
    for (int l = 1; l < 5; ++l) {
        int Hi = g.h[l - 1], Wi = g.w[l - 1];
        if (l <= 2) {   // max pool before conv2 and conv3
            const int k = l - 1;
            const long long n = (long long)g.pool(k, B2);
            if (int rc = simple_launch(kPoolName[k], lpips_pool_kernel, elementwise_grid(n), 256, st, x, v.pool[k], v.pool_arg[k], B2, Hi, Wi,
                                       kCout[k], g.ph[k], g.pw[k]))
                return rc;
            x = v.pool[k]; Hi = g.ph[k]; Wi = g.pw[k];
        }
        const ConvParams p = conv_params(x, B2, Hi, Wi, l, weights + L.w[l], weights + L.b[l], v.relu[l], g.h[l], g.w[l], false);
        if (int rc = conv(p, kConvName[l], st)) return rc;
        x = v.relu[l];
    }
    SumParams sp{};
    for (int k = 0; k < 5; ++k) {
        float *part = v.partials + (size_t)k * B * kMaxPart;
        if (int rc = dist(k, g, v.relu[k], weights + L.lin[k], part, st)) return rc;
        sp.part[k] = part; sp.nblk[k] = g.nblk(k); sp.HW[k] = g.h[k] * g.w[k];
    }
    sp.B = B; sp.out = out; sp.in_scale_ws = v.in_scale; sp.in_scale = in_scale;
    return simple_launch("lpips_sum", lpips_sum_kernel, dim3(cdiv(B, 128)), 128, st, sp);
}

extern "C" int ga_lpips_backward(int32_t B, int32_t H, int32_t W, const float *weights, void *ws, const float *g_out, float *d_in0, void *stream)
{
    using namespace ga;
    if (int rc = check_args(B, H, W, weights, ws)) return rc;
    GA_REQUIRE(g_out && d_in0, "lpips: null gradient");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Geo g(B, H, W);
    const WeightLayout L;
    GaLpipsViews v;
    carve(g, ws, &v);
    for (int k = 4; k >= 0; --k) {
        if (int rc = dnorm(k, g, v.relu[k], weights + L.lin[k], g_out, k < 4 ? v.dnext[k] : nullptr, v.dz[k], st)) return rc;
        if (k == 0) break;
        // data gradient of conv k+1 (index k): onto relu k-1 directly (conv4, conv5) or onto pool k-1's output, then un-pooled
        const bool pooled = k <= 2;
        const int Ho = pooled ? g.ph[k - 1] : g.h[k - 1], Wo = pooled ? g.pw[k - 1] : g.w[k - 1];
        float *dst = pooled ? v.dpool[k - 1] : v.dnext[k - 1];
        const ConvParams p = conv_params(v.dz[k], B, g.h[k], g.w[k], k, weights + L.wd[k], nullptr, dst, Ho, Wo, true);
        if (int rc = conv(p, kDgradName[k], st)) return rc;
        if (pooled) {
            const int j = k - 1;
            const long long n = (long long)g.map(j, B);
            if (int rc = simple_launch(kUnpoolName[j], lpips_unpool_kernel, elementwise_grid(n), 256, st, v.dpool[j], v.pool_arg[j], v.dnext[j], B,
                                       g.h[j], g.w[j], kCout[j], g.ph[j], g.pw[j]))
                return rc;
        }
    }
    const dim3 grid(cdiv((long long)((H + 3) / 4) * ((W + 3) / 4), kImgThreads), 16, B);
    return simple_launch("lpips_img_grad", lpips_img_grad_kernel, grid, kImgThreads, st, v.dz[0], weights + L.w[0], v.in_scale, H, W, g.h[0],
                         g.w[0], d_in0);
}
