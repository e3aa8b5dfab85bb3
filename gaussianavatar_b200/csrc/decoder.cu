// Feature net of GaussianAvatar stage 1 — geometry convs, UV bilinear up-sampling, ShapeDecoder MLP with training-mode
// BatchNorm — forward and backward, orchestrated on one CUDA stream.
//
// Replaces `POP_no_unet.forward(pose_featmap=None, ...)` (/root/reference model/network.py:39-83):
//   GeomConvLayers  3 x Conv2d(64,64,5,pad 2, no bias, no activation)          model/modules.py:114-137
//   uv_to_grid + F.grid_sample(bilinear, align_corners=False, zeros)            model/modules.py:745-754, network.py:61-67
//   cat([pix_feature, uv])                                                      model/network.py:69-81
//   ShapeDecoder: 14 x Conv1d(k=1), 11 x BatchNorm1d (batch statistics), Softplus, 2 x Sigmoid, skip concat at layer 5
//                                                                               model/modules.py:508-582
//
// Design (DESIGN.md §4): activations are pixel-major [M = S*S, C] fp32; each layer is ONE GEMM launch whose A-operand
// loader applies the previous layer's BatchNorm + Softplus on the fly and whose epilogue adds the bias, stores the
// pre-BN output and accumulates the per-channel batch statistics, so every hidden activation is written once and read
// once per pass.  The three heads' first layers are one N=384 GEMM.  Stage-1 inputs are identical for every frame of
// the batch (SURVEY.md §8 a-4), so the net runs once per step; `batch` only enters the unbiased running-variance update.
#include "gemm.cuh"

namespace ga {
int launch_tc_bwd(const float *dZ, const float *Y, int ldg, const float *ga, const float *m1, const float *m2, const float *mu, const float *rstd,
                  const float *Yprev, int ldp, const float *pa, const float *pb, const float *pmu, const float *prstd, const float *W, int ldw,
                  float *dW, int lddw, float *dZprev, int ldo, int mode, double *s1, double *s2, int M, int kin, int x_raw, cudaStream_t st);
int launch_tc_fwd(const float *X, int ldx, int K, const float *a, const float *b, const float *W, int ldw, const float *bias, float *Y,
                  int ldy, int accumulate, double *sum, double *sumsq, int M, cudaStream_t st, int heads = 1, size_t w_hstride = 0,
                  size_t y_hstride = 0, int v_hstride = 0);
int launch_conv_tc(int mode, const float *in, const float *w, float *out, int Hf, int round_out, cudaStream_t st);
int launch_round_tf32(const float *in, float *out, size_t n, cudaStream_t st);
namespace {

constexpr int kHeadsMinBlocks = 2;    // __launch_bounds__ min blocks per SM of the heads kernels
constexpr int kHeadsUnroll = 4;       // pixels per grid-stride trip of heads_bwd_kernel
constexpr int kHeadsGrid = kHeadsMinBlocks * kNumSMs;   // grid-stride CTAs of the heads kernels: all resident at once (<= 80 registers)
constexpr int kCg = 64;        // c_geom
constexpr int kH = 128;        // hsize
constexpr int kFeatLd = 72;    // 64 sampled + 2 uv + 6 zero pad (multiple of 8)
constexpr int kK5 = kFeatLd + kH;   // 200
constexpr int kBnCh = 5 * kH + 3 * kH + 3 * kH;   // 1408 BatchNorm channels
constexpr int kBnOff[7] = {0, 128, 256, 384, 512, 640, 1024};

struct Layout {
    int64_t gconv[3];
    int64_t w[7], b[7], gamma[7], beta[7];
    int64_t w8, b8, total;
};

Layout make_layout()
{
    Layout L;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t r = o; o += (n + 3) / 4 * 4; return r; };
    for (int i = 0; i < 3; ++i) L.gconv[i] = take(25 * kCg * kCg);
    const int kdim[7] = {kFeatLd, kH, kH, kH, kK5, kH, kH};
    const int ndim[7] = {kH, kH, kH, kH, kH, 3 * kH, 3 * kH};
    for (int l = 0; l < 7; ++l) {
        L.w[l] = take((int64_t)ndim[l] * kdim[l]);
        L.b[l] = take(ndim[l]);
        L.gamma[l] = take(ndim[l]);
        L.beta[l] = take(ndim[l]);
    }
    L.w8 = take(8 * kH);
    L.b8 = take(8);
    L.total = o;
    return L;
}

struct Workspace {
    float *F[4];          // NHWC [Hf*Wf, 64]: geo, conv1, conv2, conv3 (tensor-core path: F[0..2] hold TF32-rounded values)
    float *wr;            // [3][25*64*64] TF32-rounded copy of the conv weights (tensor-core path)
    float *dF[2];         // ping-pong gradients of the above
    float *Fp, *dFp;      // [frames][Hf*Wf, 64]: per-frame input map conv3(geo) + pose_featmap (stage 2, model/network.py:58) and its gradient
    float *feat;          // [M, 72]
    float *d_feat;        // [M, 72]
    float *Y[5];          // [M,128] pre-BN outputs of layers 1..5
    float *Y6, *Y7;       // [M,384]
    float *dZa, *dZb;     // [M,128] ping-pong
    float *dZ6, *dZ7;     // [M,384]
    double *stat;         // [4][1408]: sum, sumsq, s1, s2
    float *coef;          // [7][1408]: mean, rstd, a, b, ga, m1, m2
    size_t total;
};

Workspace carve_ws(void *buf, int S, int Hf, int frames)
{
    Carver c(buf);
    Workspace w;
    const size_t M = (size_t)frames * S * S, P = (size_t)Hf * Hf;
    for (int i = 0; i < 4; ++i) w.F[i] = c.take<float>(P * kCg);
    for (int i = 0; i < 2; ++i) w.dF[i] = c.take<float>(P * kCg);
    w.wr = c.take<float>((size_t)3 * 25 * kCg * kCg);
    w.Fp = c.take<float>(frames > 1 ? (size_t)frames * P * kCg : 4);
    w.dFp = c.take<float>(frames > 1 ? (size_t)frames * P * kCg : 4);
    w.feat = c.take<float>(M * kFeatLd);
    w.d_feat = c.take<float>(M * kFeatLd);
    for (int i = 0; i < 5; ++i) w.Y[i] = c.take<float>(M * kH);
    w.Y6 = c.take<float>(M * 3 * kH);
    w.Y7 = c.take<float>(M * 3 * kH);
    w.dZa = c.take<float>(M * kH);
    w.dZb = c.take<float>(M * kH);
    w.dZ6 = c.take<float>(M * 3 * kH);
    w.dZ7 = c.take<float>(M * 3 * kH);
    w.stat = c.take<double>(4 * kBnCh);
    w.coef = c.take<float>(7 * kBnCh);
    w.total = c.used();
    return w;
}

// ---- small kernels ---------------------------------------------------------------------------------------------

// [C, P] <-> [P, C] with C = 64 (tile transpose through shared memory)
__global__ void __launch_bounds__(256) chw_to_hwc_kernel(const float *__restrict__ in, float *__restrict__ out, int P)
{
    __shared__ float t[64][65];
    const int p0 = blockIdx.x * 64;
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int c = i / 64, p = i % 64;
        t[c][p] = (p0 + p < P) ? in[(size_t)c * P + p0 + p] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int p = i / 64, c = i % 64;
        if (p0 + p < P) out[(size_t)(p0 + p) * 64 + c] = t[c][p];
    }
}
__global__ void __launch_bounds__(256) hwc_to_chw_kernel(const float *__restrict__ in, float *__restrict__ out, int P)
{
    __shared__ float t[64][65];
    const int p0 = blockIdx.x * 64;
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int p = i / 64, c = i % 64;
        t[c][p] = (p0 + p < P) ? in[(size_t)(p0 + p) * 64 + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int c = i / 64, p = i % 64;
        if (p0 + p < P) out[(size_t)c * P + p0 + p] = t[c][p];
    }
}

// out[p][c] = in_chw[c][p] + base[p][c]: the per-frame decoder input map of stage 2, pose_featmap + geom_featmap (model/network.py:58)
__global__ void __launch_bounds__(256) chw_to_hwc_add_kernel(const float *__restrict__ in, const float *__restrict__ base, float *__restrict__ out, int P)
{
    __shared__ float t[64][65];
    const int p0 = blockIdx.x * 64;
    in += (size_t)blockIdx.y * 64 * P; out += (size_t)blockIdx.y * 64 * P;
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int c = i / 64, p = i % 64;
        t[c][p] = (p0 + p < P) ? in[(size_t)c * P + p0 + p] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int p = i / 64, c = i % 64;
        if (p0 + p < P) out[(size_t)(p0 + p) * 64 + c] = t[c][p] + base[(size_t)(p0 + p) * 64 + c];
    }
}
// out[i] = sum_f in[f][i]
__global__ void __launch_bounds__(256) sum_frames_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t n4, int frames)
{
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n4) return;
    float4 a = in[i];
    for (int f = 1; f < frames; ++f) { const float4 v = in[(size_t)f * n4 + i]; a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
    out[i] = a;
}

// Bilinear taps of F.grid_sample(align_corners=False, zeros) for query pixel (row i, col j) of an S x S UV grid over an
// Hf x Hf map — same fp32 operation order as torch: u = idx/(S-1); g = u*2-1; ix = ((g+1)*size-1)/2.
struct Taps {
    int x0, y0;
    float wx1, wy1;   // weights of (x0+1), (y0+1); 1-w for x0 / y0
};
__device__ __forceinline__ Taps make_taps(int i, int j, int S, int Hf)
{
    const float u = (float)i / (float)(S - 1), v = (float)j / (float)(S - 1);
    const float gy = u * 2.f - 1.f, gx = v * 2.f - 1.f;
    const float iy = ((gy + 1.f) * (float)Hf - 1.f) / 2.f, ix = ((gx + 1.f) * (float)Hf - 1.f) / 2.f;
    Taps t;
    const float fx = floorf(ix), fy = floorf(iy);
    t.x0 = (int)fx; t.y0 = (int)fy;
    t.wx1 = ix - fx; t.wy1 = iy - fy;
    return t;
}

// feat[m, 0:64] = bilinear(F3), feat[m,64] = row/(S-1), feat[m,65] = col/(S-1), feat[m,66:72] = 0.  16 threads / pixel.
__global__ void __launch_bounds__(256)
sample_feat_fwd_kernel(int S, int Hf, int frames, size_t frame_stride, const float *__restrict__ F, float *__restrict__ feat)
{
    const size_t gid = (size_t)blockIdx.x * 256 + threadIdx.x;
    const size_t m = gid >> 4;
    const int q = (int)(gid & 15);
    if (m >= (size_t)frames * S * S) return;
    const size_t ml = m % ((size_t)S * S);             // pixel inside its frame; the frame's map starts frame_stride floats further
    F += (m / ((size_t)S * S)) * frame_stride;
    const int i = (int)(ml / S), j = (int)(ml % S);
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (Hf == S) {
        o = *reinterpret_cast<const float4 *>(F + ml * kCg + q * 4);
    } else {
        const Taps t = make_taps(i, j, S, Hf);
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const int x = t.x0 + dx, y = t.y0 + dy;
                if (x < 0 || x >= Hf || y < 0 || y >= Hf) continue;
                const float w = (dx ? t.wx1 : 1.f - t.wx1) * (dy ? t.wy1 : 1.f - t.wy1);
                const float4 v = *reinterpret_cast<const float4 *>(F + ((size_t)y * Hf + x) * kCg + q * 4);
                o.x += w * v.x; o.y += w * v.y; o.z += w * v.z; o.w += w * v.w;
            }
    }
    *reinterpret_cast<float4 *>(feat + m * kFeatLd + q * 4) = o;
    if (q < 2) {
        float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q == 0) { e.x = (float)i / (float)(S - 1); e.y = (float)j / (float)(S - 1); }
        *reinterpret_cast<float4 *>(feat + m * kFeatLd + 64 + q * 4) = e;
    }
}

// transpose of the above: scatter d_feat[m, 0:64] into dF (pre-zeroed) with 16-byte vector reductions
__global__ void __launch_bounds__(256)
sample_feat_bwd_kernel(int S, int Hf, int frames, size_t frame_stride, const float *__restrict__ d_feat, float *__restrict__ dF)
{
    const size_t gid = (size_t)blockIdx.x * 256 + threadIdx.x;
    const size_t m = gid >> 4;
    const int q = (int)(gid & 15);
    if (m >= (size_t)frames * S * S) return;
    const size_t ml = m % ((size_t)S * S);
    dF += (m / ((size_t)S * S)) * frame_stride;
    const int i = (int)(ml / S), j = (int)(ml % S);
    const float4 g = *reinterpret_cast<const float4 *>(d_feat + m * kFeatLd + q * 4);
    if (Hf == S) {
        red_add_v4(dF + ml * kCg + q * 4, g.x, g.y, g.z, g.w);
        return;
    }
    const Taps t = make_taps(i, j, S, Hf);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const int x = t.x0 + dx, y = t.y0 + dy;
            if (x < 0 || x >= Hf || y < 0 || y >= Hf) continue;
            const float w = (dx ? t.wx1 : 1.f - t.wx1) * (dy ? t.wy1 : 1.f - t.wy1);
            red_add_v4(dF + ((size_t)y * Hf + x) * kCg + q * 4, w * g.x, w * g.y, w * g.z, w * g.w);
        }
}

// BatchNorm statistics -> folded coefficients (+ running-stat update, modules.py:530-546 / torch semantics)
__global__ void bn_finalize_fwd_kernel(int C, double count, double count_running, float eps, float momentum,
                                       const double *__restrict__ sum, const double *__restrict__ sumsq,
                                       const float *__restrict__ gamma, const float *__restrict__ beta,
                                       float *__restrict__ mean, float *__restrict__ rstd, float *__restrict__ a,
                                       float *__restrict__ b, float *__restrict__ run_mean, float *__restrict__ run_var)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const double mu = sum[c] / count;
    double var = sumsq[c] / count - mu * mu;
    if (var < 0.0) var = 0.0;
    const float rs = (float)(1.0 / sqrt(var + (double)eps));
    mean[c] = (float)mu; rstd[c] = rs;
    const float av = gamma[c] * rs;
    a[c] = av; b[c] = beta[c] - (float)mu * av;
    if (run_mean) {
        run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)mu;
        run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)(var * count_running / (count_running - 1.0));
    }
}

__global__ void bn_finalize_bwd_kernel(int C, double count, const double *__restrict__ s1, const double *__restrict__ s2,
                                       const float *__restrict__ gamma, const float *__restrict__ rstd,
                                       float *__restrict__ ga, float *__restrict__ m1, float *__restrict__ m2,
                                       float *__restrict__ d_gamma, float *__restrict__ d_beta)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    ga[c] = gamma[c] * rstd[c];
    m1[c] = (float)(s1[c] / count);
    m2[c] = (float)(s2[c] / count);
    d_gamma[c] = (float)s2[c];
    d_beta[c] = (float)s1[c];
}

// softplus(z) and sigmoid(z) from ONE exponential: e = exp(-|z|); softplus = max(z,0) + log(1+e); sigmoid = (z >= 0 ? 1 : e) / (1 + e).
// FAST (TF32 path): 3 MUFU ops (ex2, lg2, rcp); exact path: the fp32 library forms the parity tests are written against.
template <bool FAST>
__device__ __forceinline__ void softplus_sigmoid(float z, float &sp, float &sg)
{
    if (FAST) {
        const float e = __expf(-fabsf(z)), d = 1.f + e;
        sp = fmaxf(z, 0.f) + __logf(d);
        sg = __fdividef(z >= 0.f ? 1.f : e, d);
    } else {
        sp = softplus_f(z);
        sg = sigmoid_f(z);
    }
}

// Sum 8 per-lane values over the warp with 9 shuffles (recursive halving, same scheme as the rasterizer's gradient reduction):
// returns the total of value idx = 4*bit4(lane) + 2*bit3(lane) + bit2(lane), replicated over the lane's 4-lane group.
__device__ __forceinline__ float heads_reduce8(float (&v)[8], int lane)
{
    const bool h4 = lane & 16, h3 = lane & 8, h2 = lane & 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float send = h4 ? v[i] : v[i + 4]; v[i] = (h4 ? v[i + 4] : v[i]) + __shfl_xor_sync(0xffffffffu, send, 16); }
#pragma unroll
    for (int i = 0; i < 2; ++i) { const float send = h3 ? v[i] : v[i + 2]; v[i] = (h3 ? v[i + 2] : v[i]) + __shfl_xor_sync(0xffffffffu, send, 8); }
    { const float send = h2 ? v[0] : v[1]; v[0] = (h2 ? v[1] : v[0]) + __shfl_xor_sync(0xffffffffu, send, 4); }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 2);
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
    return v[0];
}


// Final 1x1 convs of the three heads (conv8 128->3, conv8N 128->1 + sigmoid, conv8SH 128->3 + sigmoid,
// modules.py:566-580) fused with the last BN + Softplus.  One warp per pixel, lane = 4 channels of each head (every
// coefficient is a thread constant; a pixel's 1.5 KB is three 512-byte warp loads), 7 dot products reduced with 9 shuffles.
template <bool FAST>
__global__ void __launch_bounds__(256, kHeadsMinBlocks)
heads_fwd_kernel(size_t M, const float *__restrict__ Y7 /*[M,384]*/, const float *__restrict__ a7, const float *__restrict__ b7,
                 const float *__restrict__ W8 /*[8,128]*/, const float *__restrict__ b8, float *__restrict__ dec /*[M,8]*/)
{
    const int lane = threadIdx.x & 31, c = lane * 4;
    float4 A[3], B[3], Wv[7];
#pragma unroll
    for (int h = 0; h < 3; ++h) { A[h] = *reinterpret_cast<const float4 *>(a7 + h * kH + c); B[h] = *reinterpret_cast<const float4 *>(b7 + h * kH + c); }
#pragma unroll
    for (int o = 0; o < 7; ++o) Wv[o] = *reinterpret_cast<const float4 *>(W8 + o * kH + c);
    const int idx = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);      // output this lane ends up holding
    const float bias = idx < 7 ? b8[idx] : 0.f;
    const size_t nwarps = (size_t)gridDim.x * 8;
    for (size_t mb = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5); mb < M; mb += 2 * nwarps) {
        float4 yy[2][3];                                                  // two pixels per trip: six 512-byte warp loads in flight
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
            for (int h = 0; h < 3; ++h)
                yy[u][h] = (mb + u * nwarps < M) ? *reinterpret_cast<const float4 *>(Y7 + (mb + u * nwarps) * 3 * kH + h * kH + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const size_t m = mb + u * nwarps;
            if (m >= M) break;
            float p[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 3; ++h) {
                const float4 y = yy[u][h];
                const float z4[4] = {fmaf(y.x, A[h].x, B[h].x), fmaf(y.y, A[h].y, B[h].y), fmaf(y.z, A[h].z, B[h].z), fmaf(y.w, A[h].w, B[h].w)};
                float x[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = FAST ? softplus_fast(z4[e]) : softplus_f(z4[e]);
                constexpr int o0[3] = {0, 3, 4}, no[3] = {3, 1, 3};
#pragma unroll
                for (int o = 0; o < 3; ++o)
                    if (o < no[h]) {
                        const float4 w = Wv[o0[h] + o];
                        p[o0[h] + o] = fmaf(x[0], w.x, fmaf(x[1], w.y, fmaf(x[2], w.z, x[3] * w.w)));
                    }
            }
            const float r = heads_reduce8(p, lane) + bias;
            if ((lane & 3) == 0) dec[m * 8 + idx] = idx < 3 ? r : (idx < 7 ? sigmoid_f(r) : 0.f);
        }
    }
}

// Backward of one head's final conv (+ sigmoid) and of the BN+Softplus feeding it.  HEAD 0: xyz (rows 0-2),
// 1: scale (row 3), 2: colour (rows 4-6).  Writes dZ7[:, head*128 ...], accumulates s1/s2 (double), dW8 rows, db8.
// One warp per pixel, lane = 4 channels: the running sums for dW8 / BatchNorm statistics are 4 x (NOUT + 2) registers.
template <int HEAD, bool FAST>
__global__ void __launch_bounds__(256, kHeadsMinBlocks)
heads_bwd_kernel(size_t M, const float *__restrict__ Y7, const float *__restrict__ a7, const float *__restrict__ b7,
                 const float *__restrict__ mu7, const float *__restrict__ rstd7, const float *__restrict__ W8,
                 const float *__restrict__ dec, const float *__restrict__ d_dec, float *__restrict__ dZ7,
                 double *__restrict__ s1, double *__restrict__ s2, float *__restrict__ dW8, float *__restrict__ db8)
{
    constexpr int NOUT = (HEAD == 1) ? 1 : 3;
    constexpr int ROW0 = (HEAD == 0) ? 0 : (HEAD == 1 ? 3 : 4);
    __shared__ float sacc[NOUT + 2][kH];
    __shared__ float sdb[NOUT];
    for (int i = threadIdx.x; i < (NOUT + 2) * kH; i += 256) sacc[i / kH][i % kH] = 0.f;
    if (threadIdx.x < NOUT) sdb[threadIdx.x] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31, c = lane * 4;
    const float4 av = *reinterpret_cast<const float4 *>(a7 + HEAD * kH + c), bv = *reinterpret_cast<const float4 *>(b7 + HEAD * kH + c);
    const float4 muv = *reinterpret_cast<const float4 *>(mu7 + HEAD * kH + c), rsv = *reinterpret_cast<const float4 *>(rstd7 + HEAD * kH + c);
    const float a_[4] = {av.x, av.y, av.z, av.w}, b_[4] = {bv.x, bv.y, bv.z, bv.w}, mu_[4] = {muv.x, muv.y, muv.z, muv.w},
                rs_[4] = {rsv.x, rsv.y, rsv.z, rsv.w};
    float w_[NOUT][4];
#pragma unroll
    for (int o = 0; o < NOUT; ++o) {
        const float4 w = *reinterpret_cast<const float4 *>(W8 + (ROW0 + o) * kH + c);
        w_[o][0] = w.x; w_[o][1] = w.y; w_[o][2] = w.z; w_[o][3] = w.w;
    }
    float aw[NOUT][4], a1[4], a2[4], adb[NOUT];
#pragma unroll
    for (int o = 0; o < NOUT; ++o) { adb[o] = 0.f; aw[o][0] = aw[o][1] = aw[o][2] = aw[o][3] = 0.f; }
#pragma unroll
    for (int e = 0; e < 4; ++e) a1[e] = a2[e] = 0.f;

    const size_t nwarps = (size_t)gridDim.x * 8;
    constexpr int U = kHeadsUnroll;                                       // pixels per trip: U 512-byte warp loads in flight
    for (size_t mb = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5); mb < M; mb += U * nwarps) {
        float4 yv[U]; float dpv[U][NOUT];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t m = mb + u * nwarps;
            const bool ok = m < M;
            yv[u] = ok ? *reinterpret_cast<const float4 *>(Y7 + m * 3 * kH + HEAD * kH + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int o = 0; o < NOUT; ++o) {                             // same address for every lane: one broadcast transaction
                const float g = ok ? d_dec[m * 8 + ROW0 + o] : 0.f;
                if (HEAD == 0) dpv[u][o] = g;                            // conv8: no output activation
                else { const float sv = ok ? dec[m * 8 + ROW0 + o] : 0.f; dpv[u][o] = g * sv * (1.f - sv); }   // sigmoid backward
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t m = mb + u * nwarps;
            if (m >= M) break;
            const float y[4] = {yv[u].x, yv[u].y, yv[u].z, yv[u].w};
            float dz[4];
#pragma unroll
            for (int o = 0; o < NOUT; ++o) adb[o] += dpv[u][o];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float z = fmaf(y[e], a_[e], b_[e]);
                float x, sg;
                softplus_sigmoid<FAST>(z, x, sg);
                float dx = 0.f;
#pragma unroll
                for (int o = 0; o < NOUT; ++o) { dx = fmaf(dpv[u][o], w_[o][e], dx); aw[o][e] = fmaf(dpv[u][o], x, aw[o][e]); }
                dz[e] = dx * sg;
                a1[e] += dz[e];
                a2[e] = fmaf(dz[e], (y[e] - mu_[e]) * rs_[e], a2[e]);
            }
            *reinterpret_cast<float4 *>(dZ7 + m * 3 * kH + HEAD * kH + c) = make_float4(dz[0], dz[1], dz[2], dz[3]);
        }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
#pragma unroll
        for (int o = 0; o < NOUT; ++o) atomicAdd(&sacc[o][c + e], aw[o][e]);
        atomicAdd(&sacc[NOUT][c + e], a1[e]);
        atomicAdd(&sacc[NOUT + 1][c + e], a2[e]);
    }
    if (lane == 0) {
#pragma unroll
        for (int o = 0; o < NOUT; ++o) atomicAdd(&sdb[o], adb[o]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kH; i += 256) {
#pragma unroll
        for (int o = 0; o < NOUT; ++o) atomicAdd(&dW8[(ROW0 + o) * kH + i], sacc[o][i]);
        atomicAdd(&s1[HEAD * kH + i], (double)sacc[NOUT][i]);
        atomicAdd(&s2[HEAD * kH + i], (double)sacc[NOUT + 1][i]);
    }
    if (threadIdx.x < NOUT) atomicAdd(&db8[ROW0 + threadIdx.x], sdb[threadIdx.x]);
}

// ---- conv loaders (5x5, 64 channels, NHWC, implicit GEMM) --------------------------------------------------------

// A'(m = pixel, k = tap*64 + ci) = In[(y + sgn*dy, x + sgn*dx), ci]; sgn = +1 forward, -1 for the data gradient
template <int BM>
struct ALoadIm2colK {
    using Frag = FragK<BM>;
    const float *In; int Hf; int sgn; int M;
    __device__ __forceinline__ void fetch(Frag &f, int m0, int k0, int tid) const
    {
        const int k = k0 + (tid & 3) * 4;
        const int tap = k >> 6, ci = k & 63;
        const int dy = sgn * (tap / 5 - 2), dx = sgn * (tap % 5 - 2);
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int m = m0 + (tid >> 2) + 64 * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < M && tap < 25) {
                const int y = m / Hf + dy, x = m % Hf + dx;
                if (y >= 0 && y < Hf && x >= 0 && x < Hf) v = *reinterpret_cast<const float4 *>(In + ((size_t)y * Hf + x) * kCg + ci);
            }
            f.v[i] = v;
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragK<BM>(S, f, tid); }
};

// A'(mg = tap*64 + ci, kg = pixel) = In[(y + dy, x + dx), ci]: direct.  Weight gradient.
template <int BM>
struct ALoadIm2colD {
    using Frag = FragD<BM>;
    const float *In; int Hf; int Mg /*1600*/, Kg /*pixels*/;
    __device__ __forceinline__ void fetch(Frag &f, int m0, int k0, int tid) const
    {
        const int c = m0 + (tid % Frag::kPerRow) * 4;
        const int tap = c >> 6, ci = c & 63;
        const int dy = tap / 5 - 2, dx = tap % 5 - 2;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int p = k0 + tid / Frag::kPerRow + Frag::kRowsPerPass * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < Kg && c < Mg) {
                const int y = p / Hf + dy, x = p % Hf + dx;
                if (y >= 0 && y < Hf && x >= 0 && x < Hf) v = *reinterpret_cast<const float4 *>(In + ((size_t)y * Hf + x) * kCg + ci);
            }
            f.v[i] = v;
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragD<BM>(S, f, tid); }
};

// B'(k = tap*64 + co, n = ci) = Wt[tap][ci][co] (co fastest): transposing.  Data gradient of the conv.
template <int BN>
struct BLoadConvDgrad {
    using Frag = FragK<BN>;
    const float *Wt;
    __device__ __forceinline__ void fetch(Frag &f, int n0, int k0, int tid) const
    {
        const int k = k0 + (tid & 3) * 4;
        const int tap = k >> 6, co = k & 63;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int n = n0 + (tid >> 2) + 64 * i;
            f.v[i] = (n < kCg && tap < 25) ? *reinterpret_cast<const float4 *>(Wt + ((size_t)tap * kCg + n) * kCg + co) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragK<BN>(S, f, tid); }
};

// ---- launch helpers --------------------------------------------------------------------------------------------
template <int BM, int BN, class AL, class BL, class EP>
int launch_gemm(const char *name, const AL &A, const BL &B, const EP &E, int Mg, int Ng, int Kg, int splits, cudaStream_t st)
{
    int kps = Kg;
    if (splits > 1) {
        kps = (cdiv(Kg, splits) + kBK - 1) / kBK * kBK;
        splits = cdiv(Kg, kps);
    } else splits = 1;
    dim3 grid(cdiv(Mg, BM), cdiv(Ng, BN), splits);
    {
        ProfScope _ps(name, st);
        gemm_kernel<BM, BN, AL, BL, EP><<<grid, kGemmThreads, 0, st>>>(A, B, E, Kg, kps);
    }
    GA_CHECK_LAUNCH(name);
    return GA_OK;
}

struct Coef {   // views into Workspace::coef
    float *mean, *rstd, *a, *b, *ga, *m1, *m2;
};
Coef coef_views(const Workspace &w)
{
    return Coef{w.coef, w.coef + kBnCh, w.coef + 2 * kBnCh, w.coef + 3 * kBnCh, w.coef + 4 * kBnCh, w.coef + 5 * kBnCh, w.coef + 6 * kBnCh};
}

int check_desc(const GaDecoderDesc *d)
{
    GA_REQUIRE(d != nullptr, "decoder desc is NULL");
    GA_REQUIRE(d->c_geom == kCg && d->hsize == kH, "only c_geom=64, hsize=128 (the reference defaults, arguments/__init__.py:101-111) are built");
    GA_REQUIRE(d->S >= 2 && d->feat_res >= 1 && d->batch >= 1, "bad decoder dims S=%d feat_res=%d batch=%d", d->S, d->feat_res, d->batch);
    GA_REQUIRE((d->S * (long long)d->S) % 4 == 0, "S*S must be a multiple of 4");
    GA_REQUIRE(d->frames >= 0 && d->frames <= 8 && (long long)(d->frames ? d->frames : 1) * d->S * d->S < (1ll << 30), "bad decoder frames=%d", d->frames);
    return GA_OK;
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_decoder_layout(const GaDecoderDesc *d, GaDecoderLayout *out)
{
    if (int rc = check_desc(d)) return rc;
    GA_REQUIRE(out, "out is NULL");
    const Layout L = make_layout();
    for (int i = 0; i < 3; ++i) out->gconv[i] = L.gconv[i];
    for (int l = 0; l < 7; ++l) { out->w[l] = L.w[l]; out->b[l] = L.b[l]; out->gamma[l] = L.gamma[l]; out->beta[l] = L.beta[l]; }
    out->w8 = L.w8; out->b8 = L.b8; out->total = L.total;
    out->bn_channels = kBnCh;
    for (int l = 0; l < 7; ++l) out->bn_offset[l] = kBnOff[l];
    return GA_OK;
}

extern "C" size_t ga_decoder_workspace_bytes(const GaDecoderDesc *d)
{
    if (check_desc(d)) return 0;
    return carve_ws(nullptr, d->S, d->feat_res, d->frames ? d->frames : 1).total;
}

extern "C" int ga_decoder_forward(const GaDecoderDesc *d, const float *params, const float *geo_nchw, const float *pose_feat_nchw,
                                  float *bn_running, void *workspace, float *dec_out, void *stream_)
{
    if (int rc = check_desc(d)) return rc;
    GA_REQUIRE(params && geo_nchw && workspace && dec_out, "NULL pointer argument");
    const int frames = d->frames ? d->frames : 1;
    GA_REQUIRE(frames == 1 || pose_feat_nchw, "frames > 1 needs the per-frame pose feature maps");
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const Layout L = make_layout();
    const Workspace w = carve_ws(workspace, d->S, d->feat_res, frames);
    const Coef cf = coef_views(w);
    const int S = d->S, Hf = d->feat_res, P = Hf * Hf;
    const int M = frames * S * S;                    // decoder rows: every frame's UV pixels (stage 1: one shared frame)

    {
        ProfScope _ps("chw_to_hwc_kernel", st);
        chw_to_hwc_kernel<<<cdiv(P, 64), 256, 0, st>>>(geo_nchw, w.F[0], P);
    }
    GA_CHECK_LAUNCH("chw_to_hwc_kernel");
    if (d->flags & GA_DECODER_TENSOR_CORES) {
        // tensor-core implicit GEMMs on TF32-rounded operands (what cuDNN computes for the reference's Conv2d): round the input and the
        // weights once; every conv but the last writes its output already rounded (it is only ever read as an MMA operand again)
        if (int rc = launch_round_tf32(w.F[0], w.F[0], (size_t)P * kCg, st)) return rc;
        for (int i = 0; i < 3; ++i)
            if (int rc = launch_round_tf32(params + L.gconv[i], w.wr + (size_t)i * 25 * kCg * kCg, (size_t)25 * kCg * kCg, st)) return rc;
        for (int i = 0; i < 3; ++i)
            if (int rc = launch_conv_tc(0, w.F[i], w.wr + (size_t)i * 25 * kCg * kCg, w.F[i + 1], Hf, i < 2, st)) return rc;
    } else {
        for (int i = 0; i < 3; ++i) {
            ALoadIm2colK<128> A{w.F[i], Hf, +1, P};
            BLoadDirect<64> B{params + L.gconv[i], kCg, kCg, 25 * kCg};
            EpiStoreStats E{w.F[i + 1], kCg, P, kCg, nullptr, nullptr, nullptr, false};
            if (int rc = launch_gemm<128, 64>("geom_conv_fwd", A, B, E, P, kCg, 25 * kCg, 1, st)) return rc;
        }
    }
    const float *Fsrc = w.F[3];
    size_t fstride = 0;
    if (pose_feat_nchw) {          // stage 2: pix_feature = pose_featmap + geom_featmap (model/network.py:58), one map per frame
        ProfScope _ps("chw_to_hwc_add_kernel", st);
        float *Fp = frames > 1 ? w.Fp : w.F[3];
        chw_to_hwc_add_kernel<<<dim3(cdiv(P, 64), frames), 256, 0, st>>>(pose_feat_nchw, w.F[3], Fp, P);
        Fsrc = Fp; fstride = frames > 1 ? (size_t)P * kCg : 0;
    }
    if (pose_feat_nchw) GA_CHECK_LAUNCH("chw_to_hwc_add_kernel");
    {
        ProfScope _ps("sample_feat_fwd_kernel", st);
        sample_feat_fwd_kernel<<<cdiv((long long)M * 16, 256), 256, 0, st>>>(S, Hf, frames, fstride, Fsrc, w.feat);
    }
    GA_CHECK_LAUNCH("sample_feat_fwd_kernel");
    GA_CHECK_CUDA(cudaMemsetAsync(w.stat, 0, sizeof(double) * 2 * kBnCh, st));

    double *sum = w.stat, *sumsq = w.stat + kBnCh;
    auto finalize = [&](int l, int C) -> int {
        const int o = kBnOff[l];
        {
            ProfScope _ps("bn_finalize_fwd_kernel", st);
            bn_finalize_fwd_kernel<<<cdiv(C, 128), 128, 0, st>>>(C, (double)M, (double)S * S * d->batch, d->bn_eps, d->bn_momentum, sum + o, sumsq + o,
                                                                 params + L.gamma[l] , params + L.beta[l], cf.mean + o, cf.rstd + o, cf.a + o, cf.b + o,
                                                                 bn_running ? bn_running + o : nullptr, bn_running ? bn_running + kBnCh + o : nullptr);
        }
        GA_CHECK_LAUNCH("bn_finalize_fwd_kernel");
        return GA_OK;
    };
    if (d->flags & GA_DECODER_TENSOR_CORES) {
        // ---- tensor-core / TF32 path: one persistent launch per 128-wide layer (mlp_tc.cu) ----
        if (int rc = launch_tc_fwd(w.feat, kFeatLd, kFeatLd, nullptr, nullptr, params + L.w[0], kFeatLd, params + L.b[0], w.Y[0], kH, 0,
                                   sum + kBnOff[0], sumsq + kBnOff[0], M, st)) return rc;
        if (int rc = finalize(0, kH)) return rc;
        for (int l = 1; l <= 3; ++l) {
            if (int rc = launch_tc_fwd(w.Y[l - 1], kH, kH, cf.a + kBnOff[l - 1], cf.b + kBnOff[l - 1], params + L.w[l], kH, params + L.b[l], w.Y[l], kH,
                                       0, sum + kBnOff[l], sumsq + kBnOff[l], M, st)) return rc;
            if (int rc = finalize(l, kH)) return rc;
        }
        // layer 5 = feat part (K=72, raw) then the x4 part accumulating on top (K=128) + bias + statistics
        if (int rc = launch_tc_fwd(w.feat, kFeatLd, kFeatLd, nullptr, nullptr, params + L.w[4], kK5, nullptr, w.Y[4], kH, 0, nullptr, nullptr, M, st)) return rc;
        if (int rc = launch_tc_fwd(w.Y[3], kH, kH, cf.a + kBnOff[3], cf.b + kBnOff[3], params + L.w[4] + kFeatLd, kK5, params + L.b[4], w.Y[4], kH, 1,
                                   sum + kBnOff[4], sumsq + kBnOff[4], M, st)) return rc;
        if (int rc = finalize(4, kH)) return rc;
        // layer 6: the three heads in one launch, whose CTAs of one tile run side by side and share the reads of layer 5's output in L2
        if (int rc = launch_tc_fwd(w.Y[4], kH, kH, cf.a + kBnOff[4], cf.b + kBnOff[4], params + L.w[5], kH, params + L.b[5], w.Y6, 3 * kH, 0,
                                   sum + kBnOff[5], sumsq + kBnOff[5], M, st, 3, (size_t)kH * kH, kH, kH)) return rc;
        if (int rc = finalize(5, 3 * kH)) return rc;
        for (int h = 0; h < 3; ++h)
            if (int rc = launch_tc_fwd(w.Y6 + h * kH, 3 * kH, kH, cf.a + kBnOff[5] + h * kH, cf.b + kBnOff[5] + h * kH,
                                       params + L.w[6] + (size_t)h * kH * kH, kH, params + L.b[6] + h * kH, w.Y7 + h * kH, 3 * kH, 0,
                                       sum + kBnOff[6] + h * kH, sumsq + kBnOff[6] + h * kH, M, st)) return rc;
    } else {
    // layer 1: feat (raw) -> Y1
    {
        ALoadConcatActK<128> A{w.feat, kFeatLd, kFeatLd, nullptr, 0, ChanAffine{nullptr, nullptr}, M, kFeatLd};
        BLoadWT<128> B{params + L.w[0], kFeatLd, kH, kFeatLd};
        EpiStoreStats E{w.Y[0], kH, M, kH, params + L.b[0], sum + kBnOff[0], sumsq + kBnOff[0], false};
        if (int rc = launch_gemm<128, 128>("mlp_fwd_l1", A, B, E, M, kH, kFeatLd, 1, st)) return rc;
        if (int rc = finalize(0, kH)) return rc;
    }
    for (int l = 1; l <= 3; ++l) {   // layers 2..4
        ALoadConcatActK<128> A{nullptr, 0, 0, w.Y[l - 1], kH, ChanAffine{cf.a + kBnOff[l - 1], cf.b + kBnOff[l - 1]}, M, kH};
        BLoadWT<128> B{params + L.w[l], kH, kH, kH};
        EpiStoreStats E{w.Y[l], kH, M, kH, params + L.b[l], sum + kBnOff[l], sumsq + kBnOff[l], false};
        if (int rc = launch_gemm<128, 128>("mlp_fwd_l2_4", A, B, E, M, kH, kH, 1, st)) return rc;
        if (int rc = finalize(l, kH)) return rc;
    }
    {   // layer 5: [feat | act(bn4(Y4))]
        ALoadConcatActK<128> A{w.feat, kFeatLd, kFeatLd, w.Y[3], kH, ChanAffine{cf.a + kBnOff[3], cf.b + kBnOff[3]}, M, kK5};
        BLoadWT<128> B{params + L.w[4], kK5, kH, kK5};
        EpiStoreStats E{w.Y[4], kH, M, kH, params + L.b[4], sum + kBnOff[4], sumsq + kBnOff[4], false};
        if (int rc = launch_gemm<128, 128>("mlp_fwd_l5", A, B, E, M, kH, kK5, 1, st)) return rc;
        if (int rc = finalize(4, kH)) return rc;
    }
    {   // layer 6 of the three heads as one N=384 GEMM
        ALoadConcatActK<128> A{nullptr, 0, 0, w.Y[4], kH, ChanAffine{cf.a + kBnOff[4], cf.b + kBnOff[4]}, M, kH};
        BLoadWT<128> B{params + L.w[5], kH, 3 * kH, kH};
        EpiStoreStats E{w.Y6, 3 * kH, M, 3 * kH, params + L.b[5], sum + kBnOff[5], sumsq + kBnOff[5], false};
        if (int rc = launch_gemm<128, 128>("mlp_fwd_l6", A, B, E, M, 3 * kH, kH, 1, st)) return rc;
        if (int rc = finalize(5, 3 * kH)) return rc;
    }
    for (int h = 0; h < 3; ++h) {   // layer 7, per head
        ALoadConcatActK<128> A{nullptr, 0, 0, w.Y6 + h * kH, 3 * kH, ChanAffine{cf.a + kBnOff[5] + h * kH, cf.b + kBnOff[5] + h * kH}, M, kH};
        BLoadWT<128> B{params + L.w[6] + (size_t)h * kH * kH, kH, kH, kH};
        EpiStoreStats E{w.Y7 + h * kH, 3 * kH, M, kH, params + L.b[6] + h * kH, sum + kBnOff[6] + h * kH, sumsq + kBnOff[6] + h * kH, false};
        if (int rc = launch_gemm<128, 128>("mlp_fwd_l7", A, B, E, M, kH, kH, 1, st)) return rc;
    }
    }
    if (int rc = finalize(6, 3 * kH)) return rc;
    {
        ProfScope _ps("heads_fwd_kernel", st);
        if (d->flags & GA_DECODER_TENSOR_CORES)
            heads_fwd_kernel<true><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + kBnOff[6], cf.b + kBnOff[6], params + L.w8, params + L.b8, dec_out);
        else
            heads_fwd_kernel<false><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + kBnOff[6], cf.b + kBnOff[6], params + L.w8, params + L.b8, dec_out);
    }
    GA_CHECK_LAUNCH("heads_fwd_kernel");
    return GA_OK;
}

extern "C" int ga_decoder_backward(const GaDecoderDesc *d, const float *params, void *workspace, const float *dec_out,
                                   const float *d_dec_out, float *d_params, float *d_geo_nchw, float *d_pose_feat_nchw, void *stream_)
{
    if (int rc = check_desc(d)) return rc;
    GA_REQUIRE(params && workspace && dec_out && d_dec_out && d_params && d_geo_nchw, "NULL pointer argument");
    const int frames = d->frames ? d->frames : 1;
    GA_REQUIRE(frames == 1 || d_pose_feat_nchw, "frames > 1 needs d_pose_feat_nchw");
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const Layout L = make_layout();
    const Workspace w = carve_ws(workspace, d->S, d->feat_res, frames);
    const Coef cf = coef_views(w);
    const int S = d->S, Hf = d->feat_res, P = Hf * Hf;
    const int M = frames * S * S;
    const int kSplit = 2 * kNumSMs;   // split-K CTAs of a 128x128 weight-gradient tile

    GA_CHECK_CUDA(cudaMemsetAsync(d_params, 0, sizeof(float) * (size_t)L.total, st));
    double *s1 = w.stat + 2 * kBnCh, *s2 = w.stat + 3 * kBnCh;
    GA_CHECK_CUDA(cudaMemsetAsync(s1, 0, sizeof(double) * 2 * kBnCh, st));

    auto finalize = [&](int l, int C) -> int {
        const int o = kBnOff[l];
        {
            ProfScope _ps("bn_finalize_bwd_kernel", st);
            bn_finalize_bwd_kernel<<<cdiv(C, 128), 128, 0, st>>>(C, (double)M, s1 + o, s2 + o, params + L.gamma[l], cf.rstd + o, cf.ga + o, cf.m1 + o,
                                                                 cf.m2 + o, d_params + L.gamma[l], d_params + L.beta[l]);
        }
        GA_CHECK_LAUNCH("bn_finalize_bwd_kernel");
        return GA_OK;
    };
    auto bwdcoef = [&](int off) { return BnBwdCoef{cf.ga + off, cf.m1 + off, cf.m2 + off, cf.mean + off, cf.rstd + off}; };

    // heads: d_dec_out -> dZ7 (+ dW8, db8)
    {
        const int o7 = kBnOff[6];
        {
            ProfScope _ps("heads_bwd_kernel<0>", st);
            if (d->flags & GA_DECODER_TENSOR_CORES)
                heads_bwd_kernel<0, true><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + o7, cf.b + o7, cf.mean + o7, cf.rstd + o7, params + L.w8,
                                                                   dec_out, d_dec_out, w.dZ7, s1 + o7, s2 + o7, d_params + L.w8, d_params + L.b8);
            else
                heads_bwd_kernel<0, false><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + o7, cf.b + o7, cf.mean + o7, cf.rstd + o7, params + L.w8,
                                                                    dec_out, d_dec_out, w.dZ7, s1 + o7, s2 + o7, d_params + L.w8, d_params + L.b8);
        }
        GA_CHECK_LAUNCH("heads_bwd_kernel<0>");
        {
            ProfScope _ps("heads_bwd_kernel<1>", st);
            if (d->flags & GA_DECODER_TENSOR_CORES)
                heads_bwd_kernel<1, true><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + o7, cf.b + o7, cf.mean + o7, cf.rstd + o7, params + L.w8,
                                                                   dec_out, d_dec_out, w.dZ7, s1 + o7, s2 + o7, d_params + L.w8, d_params + L.b8);
            else
                heads_bwd_kernel<1, false><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + o7, cf.b + o7, cf.mean + o7, cf.rstd + o7, params + L.w8,
                                                                    dec_out, d_dec_out, w.dZ7, s1 + o7, s2 + o7, d_params + L.w8, d_params + L.b8);
        }
        GA_CHECK_LAUNCH("heads_bwd_kernel<1>");
        {
            ProfScope _ps("heads_bwd_kernel<2>", st);
            if (d->flags & GA_DECODER_TENSOR_CORES)
                heads_bwd_kernel<2, true><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + o7, cf.b + o7, cf.mean + o7, cf.rstd + o7, params + L.w8,
                                                                   dec_out, d_dec_out, w.dZ7, s1 + o7, s2 + o7, d_params + L.w8, d_params + L.b8);
            else
                heads_bwd_kernel<2, false><<<kHeadsGrid, 256, 0, st>>>((size_t)M, w.Y7, cf.a + o7, cf.b + o7, cf.mean + o7, cf.rstd + o7, params + L.w8,
                                                                    dec_out, d_dec_out, w.dZ7, s1 + o7, s2 + o7, d_params + L.w8, d_params + L.b8);
        }
        GA_CHECK_LAUNCH("heads_bwd_kernel<2>");
        if (int rc = finalize(6, 3 * kH)) return rc;
    }
    float *cur = nullptr, *nxt = nullptr;
    if (d->flags & GA_DECODER_TENSOR_CORES) {
        // ---- tensor-core / TF32 path: data + weight gradient of a layer in one fused launch (mlp_tc.cu: tc_bwd_kernel) ----
        auto tc = [&](const float *dZl, const float *Yl, int ldg, int ol, const float *Yp, int ldp, int op, const float *Wl, int ldw, float *dWl,
                      float *dZp, int ldo, int mode) -> int {
            return launch_tc_bwd(dZl, Yl, ldg, cf.ga + ol, cf.m1 + ol, cf.m2 + ol, cf.mean + ol, cf.rstd + ol, Yp, ldp, cf.a + op, cf.b + op,
                                 cf.mean + op, cf.rstd + op, Wl, ldw, dWl, ldw, dZp, ldo, mode, s1 + op, s2 + op, M, kH, 0, st);
        };
        for (int h = 0; h < 3; ++h)      // layer 7 heads -> dZ6[:, h]
            if (int rc = tc(w.dZ7 + h * kH, w.Y7 + h * kH, 3 * kH, kBnOff[6] + h * kH, w.Y6 + h * kH, 3 * kH, kBnOff[5] + h * kH,
                            params + L.w[6] + (size_t)h * kH * kH, kH, d_params + L.w[6] + (size_t)h * kH * kH, w.dZ6 + h * kH, 3 * kH, 0)) return rc;
        if (int rc = finalize(5, 3 * kH)) return rc;
        for (int h = 0; h < 3; ++h)      // layer 6 heads all feed x5: raw partial sums, activation backward on the last one
            if (int rc = tc(w.dZ6 + h * kH, w.Y6 + h * kH, 3 * kH, kBnOff[5] + h * kH, w.Y[4], kH, kBnOff[4], params + L.w[5] + (size_t)h * kH * kH, kH,
                            d_params + L.w[5] + (size_t)h * kH * kH, w.dZa, kH, h == 0 ? 1 : (h == 1 ? 2 : 3))) return rc;
        if (int rc = finalize(4, kH)) return rc;
        {   // layer 5: x4 part on the tensor cores, the 72-wide feature part on the CUDA cores
            const int o5 = kBnOff[4];
            if (int rc = tc(w.dZa, w.Y[4], kH, o5, w.Y[3], kH, kBnOff[3], params + L.w[4] + kFeatLd, kK5, d_params + L.w[4] + kFeatLd, w.dZb, kH, 0)) return rc;
            // the 72-wide [features | uv] part of conv5: raw input, gradient stored into d_feat (layer 1 adds to it later)
            if (int rc = launch_tc_bwd(w.dZa, w.Y[4], kH, cf.ga + o5, cf.m1 + o5, cf.m2 + o5, cf.mean + o5, cf.rstd + o5, w.feat, kFeatLd, nullptr,
                                       nullptr, nullptr, nullptr, params + L.w[4], kK5, d_params + L.w[4], kK5, w.d_feat, kFeatLd, 1, nullptr,
                                       nullptr, M, kFeatLd, 1, st)) return rc;
            if (int rc = finalize(3, kH)) return rc;
        }
        cur = w.dZb; nxt = w.dZa;
        for (int l = 3; l >= 1; --l) {
            if (int rc = tc(cur, w.Y[l], kH, kBnOff[l], w.Y[l - 1], kH, kBnOff[l - 1], params + L.w[l], kH, d_params + L.w[l], nxt, kH, 0)) return rc;
            if (int rc = finalize(l - 1, kH)) return rc;
            float *t = cur; cur = nxt; nxt = t;
        }
    } else {
    // layer 7 (per head): wgrad, then dgrad -> dZ6
    for (int h = 0; h < 3; ++h) {
        const int o7 = kBnOff[6] + h * kH, o6 = kBnOff[5] + h * kH;
        {
            ALoadBnBwdD<128> A{w.dZ7 + h * kH, w.Y7 + h * kH, 3 * kH, bwdcoef(o7), kH, M};
            BLoadConcatActD<128> B{nullptr, 0, 0, w.Y6 + h * kH, 3 * kH, ChanAffine{cf.a + o6, cf.b + o6}, kH, M};
            EpiAtomicAdd E{d_params + L.w[6] + (size_t)h * kH * kH, kH, kH, kH};
            if (int rc = launch_gemm<128, 128>("mlp_wgrad_l7", A, B, E, kH, kH, M, kSplit, st)) return rc;
        }
        {
            ALoadBnBwdK<128> A{w.dZ7 + h * kH, w.Y7 + h * kH, 3 * kH, bwdcoef(o7), M, kH};
            BLoadDirect<128> B{params + L.w[6] + (size_t)h * kH * kH, kH, kH, kH};
            EpiDgradAct E{M, kH, 0, nullptr, 0, false, w.dZ6 + h * kH, w.Y6 + h * kH, 3 * kH, cf.a + o6, cf.b + o6, cf.mean + o6, cf.rstd + o6, s1 + o6, s2 + o6};
            if (int rc = launch_gemm<128, 128>("mlp_dgrad_l7", A, B, E, M, kH, kH, 1, st)) return rc;
        }
    }
    if (int rc = finalize(5, 3 * kH)) return rc;
    // layer 6 (N=384): wgrad, dgrad -> dZ5 (in dZa)
    {
        const int o6 = kBnOff[5], o5 = kBnOff[4];
        ALoadBnBwdD<128> A{w.dZ6, w.Y6, 3 * kH, bwdcoef(o6), 3 * kH, M};
        BLoadConcatActD<128> B{nullptr, 0, 0, w.Y[4], kH, ChanAffine{cf.a + o5, cf.b + o5}, kH, M};
        EpiAtomicAdd E{d_params + L.w[5], kH, 3 * kH, kH};
        if (int rc = launch_gemm<128, 128>("mlp_wgrad_l6", A, B, E, 3 * kH, kH, M, kSplit / 2, st)) return rc;
        ALoadBnBwdK<128> A2{w.dZ6, w.Y6, 3 * kH, bwdcoef(o6), M, 3 * kH};
        BLoadDirect<128> B2{params + L.w[5], kH, kH, 3 * kH};
        EpiDgradAct E2{M, kH, 0, nullptr, 0, false, w.dZa, w.Y[4], kH, cf.a + o5, cf.b + o5, cf.mean + o5, cf.rstd + o5, s1 + o5, s2 + o5};
        if (int rc = launch_gemm<128, 128>("mlp_dgrad_l6", A2, B2, E2, M, kH, 3 * kH, 1, st)) return rc;
        if (int rc = finalize(4, kH)) return rc;
    }
    // layer 5: dZ5 in dZa -> d_feat (store) and dZ4 (in dZb)
    {
        const int o5 = kBnOff[4], o4 = kBnOff[3];
        ALoadBnBwdD<128> A{w.dZa, w.Y[4], kH, bwdcoef(o5), kH, M};
        BLoadConcatActD<128> B{w.feat, kFeatLd, kFeatLd, w.Y[3], kH, ChanAffine{cf.a + o4, cf.b + o4}, kK5, M};
        EpiAtomicAdd E{d_params + L.w[4], kK5, kH, kK5};
        if (int rc = launch_gemm<128, 128>("mlp_wgrad_l5", A, B, E, kH, kK5, M, kSplit / 2, st)) return rc;
        ALoadBnBwdK<128> A2{w.dZa, w.Y[4], kH, bwdcoef(o5), M, kH};
        BLoadDirect<128> B2{params + L.w[4], kK5, kK5, kH};
        EpiDgradAct E2{M, kK5, kFeatLd, w.d_feat, kFeatLd, false, w.dZb, w.Y[3], kH, cf.a + o4, cf.b + o4, cf.mean + o4, cf.rstd + o4, s1 + o4, s2 + o4};
        if (int rc = launch_gemm<128, 128>("mlp_dgrad_l5", A2, B2, E2, M, kK5, kH, 1, st)) return rc;
        if (int rc = finalize(3, kH)) return rc;
    }
    // layers 4, 3, 2: dZ_l alternates dZb -> dZa -> dZb -> dZa
    cur = w.dZb; nxt = w.dZa;
    for (int l = 3; l >= 1; --l) {
        const int ol = kBnOff[l], op = kBnOff[l - 1];
        ALoadBnBwdD<128> A{cur, w.Y[l], kH, bwdcoef(ol), kH, M};
        BLoadConcatActD<128> B{nullptr, 0, 0, w.Y[l - 1], kH, ChanAffine{cf.a + op, cf.b + op}, kH, M};
        EpiAtomicAdd E{d_params + L.w[l], kH, kH, kH};
        if (int rc = launch_gemm<128, 128>("mlp_wgrad_l2_4", A, B, E, kH, kH, M, kSplit, st)) return rc;
        ALoadBnBwdK<128> A2{cur, w.Y[l], kH, bwdcoef(ol), M, kH};
        BLoadDirect<128> B2{params + L.w[l], kH, kH, kH};
        EpiDgradAct E2{M, kH, 0, nullptr, 0, false, nxt, w.Y[l - 1], kH, cf.a + op, cf.b + op, cf.mean + op, cf.rstd + op, s1 + op, s2 + op};
        if (int rc = launch_gemm<128, 128>("mlp_dgrad_l2_4", A2, B2, E2, M, kH, kH, 1, st)) return rc;
        if (int rc = finalize(l - 1, kH)) return rc;
        float *t = cur; cur = nxt; nxt = t;
    }
    }
    // layer 1: cur = dZ1
    if (d->flags & GA_DECODER_TENSOR_CORES) {
        const int o1 = kBnOff[0];
        if (int rc = launch_tc_bwd(cur, w.Y[0], kH, cf.ga + o1, cf.m1 + o1, cf.m2 + o1, cf.mean + o1, cf.rstd + o1, w.feat, kFeatLd, nullptr, nullptr,
                                   nullptr, nullptr, params + L.w[0], kFeatLd, d_params + L.w[0], kFeatLd, w.d_feat, kFeatLd, 2, nullptr, nullptr, M,
                                   kFeatLd, 1, st)) return rc;
    } else
    {
        const int o1 = kBnOff[0];
        ALoadBnBwdD<128> A{cur, w.Y[0], kH, bwdcoef(o1), kH, M};
        BLoadConcatActD<128> B{w.feat, kFeatLd, kFeatLd, nullptr, 0, ChanAffine{nullptr, nullptr}, kFeatLd, M};
        EpiAtomicAdd E{d_params + L.w[0], kFeatLd, kH, kFeatLd};
        if (int rc = launch_gemm<128, 128>("mlp_wgrad_l1", A, B, E, kH, kFeatLd, M, kSplit, st)) return rc;
        ALoadBnBwdK<128> A2{cur, w.Y[0], kH, bwdcoef(o1), M, kH};
        BLoadDirect<128> B2{params + L.w[0], kFeatLd, kFeatLd, kH};
        EpiDgradAct E2{M, kFeatLd, kFeatLd, w.d_feat, kFeatLd, true, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
        if (int rc = launch_gemm<128, 128>("mlp_dgrad_l1", A2, B2, E2, M, kFeatLd, kH, 1, st)) return rc;
    }
    // up-sampling backward, then the three convs
    float *dsink = frames > 1 ? w.dFp : w.dF[0];
    GA_CHECK_CUDA(cudaMemsetAsync(dsink, 0, sizeof(float) * (size_t)frames * P * kCg, st));
    {
        ProfScope _ps("sample_feat_bwd_kernel", st);
        sample_feat_bwd_kernel<<<cdiv((long long)M * 16, 256), 256, 0, st>>>(S, Hf, frames, frames > 1 ? (size_t)P * kCg : 0, w.d_feat, dsink);
    }
    GA_CHECK_LAUNCH("sample_feat_bwd_kernel");
    if (d_pose_feat_nchw) {        // d pose_featmap[f] = d pix[f] (NCHW); d geom_featmap = sum over the frames
        for (int f = 0; f < frames; ++f) {
            ProfScope _ps("hwc_to_chw_kernel", st);
            hwc_to_chw_kernel<<<cdiv(P, 64), 256, 0, st>>>(dsink + (size_t)f * P * kCg, d_pose_feat_nchw + (size_t)f * P * kCg, P);
            GA_CHECK_LAUNCH("hwc_to_chw_kernel");
        }
    }
    if (frames > 1) {
        ProfScope _ps("sum_frames_kernel", st);
        sum_frames_kernel<<<cdiv((long long)P * kCg / 4, 256), 256, 0, st>>>(reinterpret_cast<const float4 *>(w.dFp), reinterpret_cast<float4 *>(w.dF[0]),
                                                                            (size_t)P * kCg / 4, frames);
    }
    if (frames > 1) GA_CHECK_LAUNCH("sum_frames_kernel");
    float *dcur = w.dF[0], *dnxt = w.dF[1];
    if (d->flags & GA_DECODER_TENSOR_CORES) {
        // the forward pass left F[0..2] and the weight copy TF32-rounded; the up-sampling gradient is rounded in place (it only
        // feeds MMAs), every data gradient but the last is written rounded
        if (int rc = launch_round_tf32(dcur, dcur, (size_t)P * kCg, st)) return rc;
        for (int i = 2; i >= 0; --i) {
            if (int rc = launch_conv_tc(2, w.F[i], dcur, d_params + L.gconv[i], Hf, 0, st)) return rc;
            if (int rc = launch_conv_tc(1, dcur, w.wr + (size_t)i * 25 * kCg * kCg, dnxt, Hf, i > 0, st)) return rc;
            float *t = dcur; dcur = dnxt; dnxt = t;
        }
    } else
    for (int i = 2; i >= 0; --i) {
        {
            ALoadIm2colD<128> A{w.F[i], Hf, 25 * kCg, P};
            BLoadDirect<64> B{dcur, kCg, kCg, P};
            EpiAtomicAdd E{d_params + L.gconv[i], kCg, 25 * kCg, kCg};
            if (int rc = launch_gemm<128, 64>("geom_conv_wgrad", A, B, E, 25 * kCg, kCg, P, 24, st)) return rc;
        }
        {
            ALoadIm2colK<128> A{dcur, Hf, -1, P};
            BLoadConvDgrad<64> B{params + L.gconv[i]};
            EpiStoreStats E{dnxt, kCg, P, kCg, nullptr, nullptr, nullptr, false};
            if (int rc = launch_gemm<128, 64>("geom_conv_dgrad", A, B, E, P, kCg, 25 * kCg, 1, st)) return rc;
        }
        float *t = dcur; dcur = dnxt; dnxt = t;
    }
    {
        ProfScope _ps("hwc_to_chw_kernel", st);
        hwc_to_chw_kernel<<<cdiv(P, 64), 256, 0, st>>>(dcur, d_geo_nchw, P);
    }
    GA_CHECK_LAUNCH("hwc_to_chw_kernel");
    return GA_OK;
}

// Addresses of every workspace buffer (device pointers; nothing is copied and the device is not touched).
extern "C" int ga_decoder_views(const GaDecoderDesc *d, void *workspace, GaDecoderViews *out)
{
    if (int rc = check_desc(d)) return rc;
    GA_REQUIRE(workspace && out, "NULL pointer argument");
    const Workspace w = carve_ws(workspace, d->S, d->feat_res, d->frames ? d->frames : 1);
    for (int i = 0; i < 4; ++i) out->F[i] = w.F[i];
    out->wr = w.wr;
    for (int i = 0; i < 2; ++i) out->dF[i] = w.dF[i];
    out->Fp = w.Fp; out->dFp = w.dFp;
    out->feat = w.feat; out->d_feat = w.d_feat;
    for (int i = 0; i < 5; ++i) out->Y[i] = w.Y[i];
    out->Y6 = w.Y6; out->Y7 = w.Y7;
    out->dZa = w.dZa; out->dZb = w.dZb; out->dZ6 = w.dZ6; out->dZ7 = w.dZ7;
    out->stat = w.stat;
    out->coef = w.coef;
    return GA_OK;
}
