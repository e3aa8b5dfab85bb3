// The geometry net's 5x5 convolutions (GeomConvLayers, model/modules.py:122-137: three 64->64 convs, padding 2, no bias, no
// activation) as implicit GEMMs on the tensor cores (mma.sync m16n8k8 TF32, fp32 accumulators in registers; tc_common.cuh).
//
//   mode 0  forward        Y [px][co]      = sum_{tap,ci} X [px + tap][ci] * W[tap][ci][co]
//   mode 1  data gradient  dX[px][ci]      = sum_{tap,co} dY[px - tap][co] * W[tap][ci][co]
//   mode 2  weight grad.   dW[tap][ci][co] += sum_px      X [px + tap][ci] * dY[px][co]
//
// Feature maps are NHWC [P = Hf*Hf][64] fp32 whose values are already rounded to TF32 (round_tf32_kernel, or the
// producing conv's epilogue), so operands can travel global -> shared memory with cp.async (16-byte pieces, zero-fill for the
// padding, no registers) straight into the swizzled images the fragments are read from:
//   modes 0/1: one CTA per 128 consecutive pixels; 50 K-steps (tap x 32-channel half); A = im2col rows, K-major 128 B swizzle;
//              B = W[tap][ci half][64 co] pixel-major (mode 0) or W[tap][64 ci][co half] K-major (mode 1)
//   mode 2   : one CTA per (pair of taps, pixel split); K = pixel (32 per step); A = the two taps' shifted X (M = 2 x 64 ci),
//              B = dY, both pixel-major, consumed as they lie
// Pipeline: every one of the 8 warps copies its pieces kDepth steps ahead over an 8-stage ring, then multiplies its 16 rows of the
// 128 x 64 output tile; one block barrier per step.  The accumulators leave the registers once at the end.
#include "common.cuh"
#include "tc_common.cuh"

namespace ga {
namespace {

using namespace tc;

constexpr int kC = 64, kTaps = 25;
constexpr int kCStages = 8;
constexpr int kABytes = 16384, kBBytes = 8192, kCStageBytes = kABytes + kBBytes;
constexpr int kDepth = 6;                       // steps of cp.async groups in flight (a stage is refilled 2 steps after it was read)
constexpr int kConvThreads = 8 * 32;
constexpr int kTapPairs = 13;
static_assert(kDepth + 2 <= kCStages, "a stage must not be refilled while a warp may still read it");

struct ConvParams {
    const float *in;       // modes 0, 2: X; mode 1: dY          [P][64], TF32-rounded
    const float *w;        // modes 0, 1: W [25][64 ci][64 co] TF32-rounded; mode 2: dY [P][64] TF32-rounded
    float *out;            // modes 0, 1: [P][64]; mode 2: dW [25][64][64] (accumulated with vector reductions)
    int Hf, P, round_out, nsplit;
};

struct alignas(1024) ConvSmem {
    unsigned char st[kCStages][kCStageBytes];
};

__device__ __forceinline__ float round_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }

template <int MODE>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_tc_kernel(const ConvParams p)
{
    extern __shared__ unsigned char smem_raw[];
    ConvSmem &sm = *reinterpret_cast<ConvSmem *>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t4 = lane & 3;
    const int Hf = p.Hf, P = p.P;

    // work of this CTA
    int nst, m0 = 0, tpair = 0, z = 0;
    if (MODE == 2) {
        tpair = blockIdx.x % kTapPairs; z = blockIdx.x / kTapPairs;
        const int nchunk = (P + 31) / 32;
        nst = z < nchunk ? (nchunk - z + p.nsplit - 1) / p.nsplit : 0;
        if (nst == 0) return;                                    // uniform for the CTA, before any barrier
    } else {
        m0 = blockIdx.x * 128;
        nst = 2 * kTaps;
    }

    // ================================ copies ================================
    const int u = tid & 7, rg = tid >> 3;                        // 16-byte unit, row group (0..31)
    int py[4], px[4]; bool pv[4];
    if (MODE != 2) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { const int m = m0 + rg + 32 * i; pv[i] = m < P; py[i] = m / Hf; px[i] = m % Hf; }
    }
    const uint32_t a_off = (uint32_t)rg * 128u + (uint32_t)((u ^ (rg & 7)) << 4);          // K-major A: + i * 4096  (modes 0, 1)
    const uint32_t a_off_mn = mn_unit(rg, u);                                                 // pixel-major A: + chunk * 4096 (mode 2)
    // B tile: unit v (0..15) of row kk = tid >> 4 (+16 per pass) for the 256-byte rows, or unit u of row rg (+32) for 128-byte rows
    const int v = tid & 15, kk = tid >> 4;
    const uint32_t b_off_mn = (uint32_t)(v >> 3) * 4096u + mn_unit(kk, v & 7);              // + i2 * 16 * 128 (kk & 3 unchanged)
    const uint32_t b_off_k = (uint32_t)rg * 128u + (uint32_t)((u ^ (rg & 7)) << 4);         // + i2 * 4096
    const uint32_t st0 = smem_u32(sm.st[0]);

    auto issue = [&](int q) {
        if (q < nst) {
            const uint32_t sa = st0 + (uint32_t)(q % kCStages) * kCStageBytes, sb = sa + kABytes;
            if (MODE != 2) {
                const int t = q >> 1, h = q & 1;
                const int dy = (MODE == 0 ? 1 : -1) * (t / 5 - 2), dx = (MODE == 0 ? 1 : -1) * (t % 5 - 2);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int yy = py[i] + dy, xx = px[i] + dx;
                    const bool ok = pv[i] && (unsigned)yy < (unsigned)Hf && (unsigned)xx < (unsigned)Hf;
                    const float *src = p.in + ((size_t)(ok ? yy * Hf + xx : 0) * kC + h * 32 + u * 4);
                    cp_async16(sa + a_off + i * 4096u, src, ok);
                }
                if (MODE == 0) {
#pragma unroll
                    for (int i2 = 0; i2 < 2; ++i2)
                        cp_async16_full(sb + b_off_mn + i2 * 2048u, p.w + ((size_t)(t * kC + h * 32 + kk + 16 * i2) * kC + v * 4));
                } else {
#pragma unroll
                    for (int i2 = 0; i2 < 2; ++i2)
                        cp_async16_full(sb + b_off_k + i2 * 4096u, p.w + ((size_t)(t * kC + rg + 32 * i2) * kC + h * 32 + u * 4));
                }
            } else {
                const int pxl0 = (z + q * p.nsplit) * 32;                 // first pixel of this step's 32-pixel chunk
                const int m = pxl0 + rg;
                const bool mv = m < P;
                const int y = m / Hf, x = m % Hf;
#pragma unroll
                for (int i = 0; i < 4; ++i) {                           // A chunk i: tap 2 tpair + (i >> 1), channel half i & 1
                    const int t = 2 * tpair + (i >> 1);
                    const int yy = y + t / 5 - 2, xx = x + t % 5 - 2;
                    const bool ok = mv && t < kTaps && (unsigned)yy < (unsigned)Hf && (unsigned)xx < (unsigned)Hf;
                    const float *src = p.in + ((size_t)(ok ? yy * Hf + xx : 0) * kC + (i & 1) * 32 + u * 4);
                    cp_async16(sa + a_off_mn + i * 4096u, src, ok);
                }
#pragma unroll
                for (int i2 = 0; i2 < 2; ++i2) {                         // B = dY rows (pixels) kk + 16 i2, 64 channels
                    const int mb = pxl0 + kk + 16 * i2;
                    const bool ok = mb < P;
                    cp_async16(sb + b_off_mn + i2 * 2048u, p.w + ((size_t)(ok ? mb : 0) * kC + v * 4), ok);
                }
            }
        }
        cp_async_commit();                                      // one group per step, empty past the end: the wait count stays uniform
    };

    for (int q = 0; q < kDepth; ++q) issue(q);
    float acc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
    const int mr = 16 * warp + g;                                // this lane's output rows: mr, mr + 8
    for (int q = 0; q < nst; ++q) {
        cp_async_wait<kDepth - 1>();                             // this thread's pieces of step q have landed ...
        __syncthreads();                                         // ... and everybody's; every warp is done with step q - 1
        issue(q + kDepth);
        const uint32_t sa = st0 + (uint32_t)(q % kCStages) * kCStageBytes, sb = sa + kABytes;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const int k = 8 * ks + t4;
            uint32_t a[4];
            if (MODE == 2) {
                a[0] = lds32(sa + mnmajor_off(k, mr, 4096)); a[1] = lds32(sa + mnmajor_off(k, mr + 8, 4096));
                a[2] = lds32(sa + mnmajor_off(k + 4, mr, 4096)); a[3] = lds32(sa + mnmajor_off(k + 4, mr + 8, 4096));
            } else {
                a[0] = lds32(sa + kmajor_off(mr, k, 0)); a[1] = lds32(sa + kmajor_off(mr + 8, k, 0));
                a[2] = lds32(sa + kmajor_off(mr, k + 4, 0)); a[3] = lds32(sa + kmajor_off(mr + 8, k + 4, 0));
            }
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int n = 8 * nt + g;
                uint32_t b0, b1;
                if (MODE == 1) { b0 = lds32(sb + kmajor_off(n, k, 0)); b1 = lds32(sb + kmajor_off(n, k + 4, 0)); }
                else { b0 = lds32(sb + mnmajor_off(k, n, 4096)); b1 = lds32(sb + mnmajor_off(k + 4, n, 4096)); }
                mma_tf32(acc[nt], a, b0, b1);
            }
        }
    }
    cp_async_wait<0>();

    // ================================ epilogue: rows mr, mr + 8; columns 8 nt + 2 t4, + 1 ================================
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = mr + 8 * h;
        if (MODE != 2) {
            const int m = m0 + row;
            if (m < P) {
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    float2 o = make_float2(acc[nt][2 * h], acc[nt][2 * h + 1]);
                    if (p.round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); }
                    *reinterpret_cast<float2 *>(p.out + (size_t)m * kC + 8 * nt + 2 * t4) = o;
                }
            }
        } else {
            const int t = 2 * tpair + (row >> 6), ci = row & 63;
            if (t < kTaps) {
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
                    red_add_v2(p.out + ((size_t)(t * kC + ci) * kC + 8 * nt + 2 * t4), acc[nt][2 * h], acc[nt][2 * h + 1]);
            }
        }
    }
}

__global__ void __launch_bounds__(256) round_tf32_kernel(const float *__restrict__ in, float *__restrict__ out, size_t n4)
{
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n4) return;
    float4 v = reinterpret_cast<const float4 *>(in)[i];
    v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w);
    reinterpret_cast<float4 *>(out)[i] = v;
}

template <int MODE>
int launch_mode(const ConvParams &p, int grid, const char *name, cudaStream_t st)
{
    static PerDeviceOnce attr_set;
    if (attr_set.first()) {
        GA_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ConvSmem) + 1024));
    }
    {
        ProfScope _ps(name, st);
        conv_tc_kernel<MODE><<<grid, kConvThreads, sizeof(ConvSmem) + 1024, st>>>(p);
    }
    GA_CHECK_LAUNCH(name);
    return GA_OK;
}

}  // namespace

// in-place allowed (in == out); n must be a multiple of 4 and the pointers 16-byte aligned
int launch_round_tf32(const float *in, float *out, size_t n, cudaStream_t st)
{
    GA_REQUIRE(n % 4 == 0, "round_tf32: length must be a multiple of 4");
    if (n == 0) return GA_OK;
    {
        ProfScope _ps("round_tf32_kernel", st);
        round_tf32_kernel<<<(unsigned)cdiv((long long)(n / 4), 256), 256, 0, st>>>(in, out, n / 4);
    }
    GA_CHECK_LAUNCH("round_tf32_kernel");
    return GA_OK;
}

// mode 0: out[P][64] = conv(in, w); mode 1: out = conv_transpose-style data gradient of `in` = dY; mode 2: out (dW) += wgrad(in = X, w = dY)
int launch_conv_tc(int mode, const float *in, const float *w, float *out, int Hf, int round_out, cudaStream_t st)
{
    GA_REQUIRE(mode >= 0 && mode <= 2 && in && w && out && Hf > 0, "tensor-core conv: bad arguments");
    const int P = Hf * Hf;
    ConvParams p{in, w, out, Hf, P, round_out, 1};
    if (mode == 2) {
        const int nchunk = cdiv(P, 32);
        const int split = num_sms() / kTapPairs;                 // 13 tap pairs x 10 pixel splits = 130 CTAs on 132 SMs
        p.nsplit = nchunk < split ? nchunk : split;
        return launch_mode<2>(p, kTapPairs * p.nsplit, "geom_conv_tc_wgrad", st);
    }
    const int tiles = cdiv(P, 128);
    return mode == 0 ? launch_mode<0>(p, tiles, "geom_conv_tc_fwd", st) : launch_mode<1>(p, tiles, "geom_conv_tc_dgrad", st);
}

}  // namespace ga

// Unit-test / building-block entries (TF32-rounded operands in, see the file header).
extern "C" int ga_tc_conv5x5(int32_t mode, int32_t Hf, const float *in, const float *w, float *out, int32_t round_out, void *stream)
{
    return ga::launch_conv_tc(mode, in, w, out, Hf, round_out, static_cast<cudaStream_t>(stream));
}
extern "C" int ga_round_tf32(const float *in, float *out, int64_t n, void *stream)
{
    GA_REQUIRE(in && out && n >= 0, "bad arguments");
    return ga::launch_round_tf32(in, out, (size_t)n, static_cast<cudaStream_t>(stream));
}
