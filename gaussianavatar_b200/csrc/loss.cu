// Fused image loss: L1 + SSIM (11x11 Gaussian window, sigma 1.5, zero padding), forward and backward.
//
// Replaces `l1_loss_w(image, gt)` and `ssim(image, gt)` (/root/reference utils/loss_utils.py:7-8,23-53; used at
// train.py:74-75): the reference runs 5 depthwise 11x11 convolutions + ~15 element-wise kernels forward and again
// backward over [B,3,H,W]; here one forward kernel blurs the five moment images separably in shared memory, evaluates
// the SSIM map and the L1 term, block-reduces both sums and keeps three partial-derivative maps; one backward kernel
// blurs those maps and emits dL/dimage directly in the [B,3,H,W] layout the rasterizer backward consumes.
#include "common.cuh"

namespace ga {
namespace {

constexpr int kWin = 11, kHalo = 5;
constexpr int kTX = 32, kTY = 16;                 // output tile
constexpr int kSX = kTX + 2 * kHalo, kSY = kTY + 2 * kHalo;   // 42 x 26 staged region

__constant__ float c_gauss[kWin];

void gauss_host(float *g)
{
    // utils/loss_utils.py:13-15: exp(-(x - 5)^2 / (2 * 1.5^2)) normalised, evaluated in double then narrowed like torch.Tensor([...])
    double v[kWin], s = 0.0;
    for (int i = 0; i < kWin; ++i) { v[i] = exp(-(double)((i - kHalo) * (i - kHalo)) / (2.0 * 1.5 * 1.5)); }
    float f[kWin]; float fs = 0.f;
    for (int i = 0; i < kWin; ++i) { f[i] = (float)v[i]; fs += f[i]; s += v[i]; }
    for (int i = 0; i < kWin; ++i) g[i] = f[i] / fs;
    (void)s;
}

// grid: (ceil(W/32), ceil(H/16), B*3); block: 32 x 16
__global__ void __launch_bounds__(kTX * kTY)
ssim_l1_fwd_kernel(int H, int W, const float *__restrict__ img, const float *__restrict__ gt, float *__restrict__ dm_dmu1,
                   float *__restrict__ dm_ds1, float *__restrict__ dm_ds12, double *__restrict__ acc /*[2]: ssim sum, l1 sum*/)
{
    __shared__ float sA[kSY][kSX + 1], sB[kSY][kSX + 1];
    __shared__ float sH[5][kSY][kTX + 1];
    __shared__ float sred[2][kTX * kTY / 32];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTX + tx;
    const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY;
    const size_t plane = (size_t)blockIdx.z * H * W;
    bool same = true;
    for (int i = tid; i < kSY * kSX; i += kTX * kTY) {
        const int ly = i / kSX, lx = i % kSX;
        const int y = y0 + ly - kHalo, x = x0 + lx - kHalo;
        float a = 0.f, b = 0.f;
        if (x >= 0 && x < W && y >= 0 && y < H) { a = img[plane + (size_t)y * W + x]; b = gt[plane + (size_t)y * W + x]; }
        sA[ly][lx] = a; sB[ly][lx] = b;
        same = same && (a == b);
    }
    // A tile whose whole window support shows image == target (the white background of GaussianAvatar's frames: most of the image)
    // has SSIM == 1 and L1 == 0 at every pixel, and its three derivative maps are zero up to the round-off of terms that cancel
    // (2 mu / C - 2 mu / C): write exact zeros and skip the 11x11 blurs.
    if (__syncthreads_and(same)) {
        const int x = x0 + tx, y = y0 + ty;
        float one = 0.f;
        if (x < W && y < H) {
            const size_t p = plane + (size_t)y * W + x;
            dm_dmu1[p] = 0.f; dm_ds1[p] = 0.f; dm_ds12[p] = 0.f;
            one = 1.f;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) one += __shfl_xor_sync(0xffffffffu, one, o);
        if ((tid & 31) == 0) sred[0][tid >> 5] = one;
        __syncthreads();
        if (tid == 0) {
            float sum = 0.f;
            for (int i = 0; i < kTX * kTY / 32; ++i) sum += sred[0][i];
            atomicAdd(&acc[0], (double)sum);
        }
        return;
    }
    // horizontal pass over all staged rows
    for (int i = tid; i < kSY * kTX; i += kTX * kTY) {
        const int ly = i / kTX, lx = i % kTX;
        float m1 = 0.f, m2 = 0.f, xx = 0.f, yy = 0.f, xy = 0.f;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const float w = c_gauss[k], a = sA[ly][lx + k], b = sB[ly][lx + k];
            m1 = fmaf(w, a, m1); m2 = fmaf(w, b, m2); xx = fmaf(w, a * a, xx); yy = fmaf(w, b * b, yy); xy = fmaf(w, a * b, xy);
        }
        sH[0][ly][lx] = m1; sH[1][ly][lx] = m2; sH[2][ly][lx] = xx; sH[3][ly][lx] = yy; sH[4][ly][lx] = xy;
    }
    __syncthreads();
    float mu1 = 0.f, mu2 = 0.f, xx = 0.f, yy = 0.f, xy = 0.f;
#pragma unroll
    for (int k = 0; k < kWin; ++k) {
        const float w = c_gauss[k];
        mu1 = fmaf(w, sH[0][ty + k][tx], mu1); mu2 = fmaf(w, sH[1][ty + k][tx], mu2);
        xx = fmaf(w, sH[2][ty + k][tx], xx); yy = fmaf(w, sH[3][ty + k][tx], yy); xy = fmaf(w, sH[4][ty + k][tx], xy);
    }
    const int x = x0 + tx, y = y0 + ty;
    float ssim_v = 0.f, l1_v = 0.f;
    if (x < W && y < H) {
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
        const float s1 = xx - mu1_sq, s2 = yy - mu2_sq, s12 = xy - mu12;
        const float A = 2.f * mu12 + C1, Bv = 2.f * s12 + C2, Cc = mu1_sq + mu2_sq + C1, D = s1 + s2 + C2;
        ssim_v = (A * Bv) / (Cc * D);
        const float a = sA[ty + kHalo][tx + kHalo], b = sB[ty + kHalo][tx + kHalo];
        l1_v = fabsf(a - b);
        const size_t p = plane + (size_t)y * W + x;
        dm_dmu1[p] = (mu2 * 2.f * Bv) / (Cc * D) - (mu2 * 2.f * A) / (Cc * D) - (mu1 * 2.f * A * Bv) / (Cc * Cc * D) + (mu1 * 2.f * A * Bv) / (Cc * D * D);
        dm_ds1[p] = (-A * Bv) / (Cc * D * D);
        dm_ds12[p] = (2.f * A) / (Cc * D);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { ssim_v += __shfl_xor_sync(0xffffffffu, ssim_v, o); l1_v += __shfl_xor_sync(0xffffffffu, l1_v, o); }
    if ((tid & 31) == 0) { sred[0][tid >> 5] = ssim_v; sred[1][tid >> 5] = l1_v; }
    __syncthreads();
    if (tid == 0) {
        float s = 0.f, l = 0.f;
        for (int i = 0; i < kTX * kTY / 32; ++i) { s += sred[0][i]; l += sred[1][i]; }
        atomicAdd(&acc[0], (double)s);
        atomicAdd(&acc[1], (double)l);
    }
}

// d loss / d img = cl1 * sign(img - gt) + cssim * (blur(dm_dmu1) + 2 img blur(dm_ds1) + gt blur(dm_ds12)),
// where cl1 = g * w_l1 / Npix and cssim = g * w_ssim / Npix are read from `coef` (device, written by the host wrapper's
// tiny scale kernel so that the upstream gradient never needs a host round trip).
__global__ void __launch_bounds__(kTX * kTY)
ssim_l1_bwd_kernel(int H, int W, const float *__restrict__ img, const float *__restrict__ gt, const float *__restrict__ dm_dmu1,
                   const float *__restrict__ dm_ds1, const float *__restrict__ dm_ds12, const float *__restrict__ coef /*[2]*/,
                   float *__restrict__ d_img)
{
    __shared__ float sM[3][kSY][kSX + 1];
    __shared__ float sH[3][kSY][kTX + 1];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTX + tx;
    const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY;
    const size_t plane = (size_t)blockIdx.z * H * W;
    bool zero = true;
    for (int i = tid; i < kSY * kSX; i += kTX * kTY) {
        const int ly = i / kSX, lx = i % kSX;
        const int y = y0 + ly - kHalo, x = x0 + lx - kHalo;
        float a = 0.f, b = 0.f, c = 0.f;
        if (x >= 0 && x < W && y >= 0 && y < H) {
            const size_t p = plane + (size_t)y * W + x;
            a = dm_dmu1[p]; b = dm_ds1[p]; c = dm_ds12[p];
        }
        sM[0][ly][lx] = a; sM[1][ly][lx] = b; sM[2][ly][lx] = c;
        zero = zero && (a == 0.f) && (b == 0.f) && (c == 0.f);
    }
    // all three derivative maps vanish over the window support (background tiles, see the forward): only the L1 term is left
    if (__syncthreads_and(zero)) {
        const int x = x0 + tx, y = y0 + ty;
        if (x < W && y < H) {
            const size_t p = plane + (size_t)y * W + x;
            const float d = img[p] - gt[p];
            d_img[p] = coef[0] * ((d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f));
        }
        return;
    }
    for (int i = tid; i < kSY * kTX; i += kTX * kTY) {
        const int ly = i / kTX, lx = i % kTX;
        float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const float w = c_gauss[k];
            a = fmaf(w, sM[0][ly][lx + k], a); b = fmaf(w, sM[1][ly][lx + k], b); c = fmaf(w, sM[2][ly][lx + k], c);
        }
        sH[0][ly][lx] = a; sH[1][ly][lx] = b; sH[2][ly][lx] = c;
    }
    __syncthreads();
    float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
    for (int k = 0; k < kWin; ++k) {
        const float w = c_gauss[k];
        a = fmaf(w, sH[0][ty + k][tx], a); b = fmaf(w, sH[1][ty + k][tx], b); c = fmaf(w, sH[2][ty + k][tx], c);
    }
    const int x = x0 + tx, y = y0 + ty;
    if (x < W && y < H) {
        const size_t p = plane + (size_t)y * W + x;
        const float iv = img[p], gv = gt[p];
        const float d = iv - gv;
        const float sgn = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
        d_img[p] = coef[0] * sgn + coef[1] * (a + 2.f * iv * b + gv * c);
    }
}

// out[0] = w_l1 * l1_mean + w_ssim * (1 - ssim_mean); out[1] = ssim_mean; out[2] = l1_mean
__global__ void loss_finalize_kernel(const double *__restrict__ acc, double inv_n, float w_l1, float w_ssim, float *__restrict__ out)
{
    const double s = acc[0] * inv_n, l = acc[1] * inv_n;
    out[0] = (float)(w_l1 * l + w_ssim * (1.0 - s));
    out[1] = (float)s;
    out[2] = (float)l;
}

// coef[0] = g * w_l1 / n ; coef[1] = -g * w_ssim / n   (d(1 - ssim)/d ssim = -1)
__global__ void loss_coef_kernel(const float *__restrict__ g, float w_l1, float w_ssim, float inv_n, float *__restrict__ coef)
{
    const float gv = g ? g[0] : 1.f;
    coef[0] = gv * w_l1 * inv_n;
    coef[1] = -gv * w_ssim * inv_n;
}

bool g_gauss_ready[64] = {};      // __constant__ memory is per device: one flag per device ordinal
int ensure_gauss()
{
    int dev = 0;
    GA_CHECK_CUDA(cudaGetDevice(&dev));
    GA_REQUIRE(dev >= 0 && dev < 64, "device ordinal %d out of range", dev);
    if (g_gauss_ready[dev]) return GA_OK;
    float g[kWin];
    gauss_host(g);
    GA_CHECK_CUDA(cudaMemcpyToSymbol(c_gauss, g, sizeof(g)));
    g_gauss_ready[dev] = true;
    return GA_OK;
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" size_t ga_loss_workspace_bytes(int32_t B, int32_t H, int32_t W)
{
    const size_t n = (size_t)B * 3 * H * W;
    return align_up(3 * n * sizeof(float)) + align_up(2 * sizeof(double)) + align_up(4 * sizeof(float));
}

extern "C" int ga_loss_forward(int32_t B, int32_t H, int32_t W, const float *image, const float *gt, float w_l1, float w_ssim,
                               void *workspace, float *out3, void *stream_)
{
    GA_REQUIRE(B > 0 && H > 0 && W > 0, "bad loss dims B=%d H=%d W=%d", B, H, W);
    GA_REQUIRE(image && gt && workspace && out3, "NULL pointer argument");
    if (int rc = ensure_gauss()) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const size_t n = (size_t)B * 3 * H * W;
    Carver c(workspace);
    float *maps = c.take<float>(3 * n);
    double *acc = c.take<double>(2);
    GA_CHECK_CUDA(cudaMemsetAsync(acc, 0, 2 * sizeof(double), st));
    dim3 grid(cdiv(W, kTX), cdiv(H, kTY), B * 3), block(kTX, kTY);
    { ProfScope _ps("ssim_l1_fwd_kernel", st); ssim_l1_fwd_kernel<<<grid, block, 0, st>>>(H, W, image, gt, maps, maps + n, maps + 2 * n, acc); }
    GA_CHECK_LAUNCH("ssim_l1_fwd_kernel");
    { ProfScope _ps("loss_finalize_kernel", st); loss_finalize_kernel<<<1, 1, 0, st>>>(acc, 1.0 / (double)n, w_l1, w_ssim, out3); }
    GA_CHECK_LAUNCH("loss_finalize_kernel");
    return GA_OK;
}

extern "C" int ga_loss_backward(int32_t B, int32_t H, int32_t W, const float *image, const float *gt, float w_l1, float w_ssim,
                                const float *grad_out /*device scalar or NULL (=1)*/, void *workspace, float *d_image, void *stream_)
{
    GA_REQUIRE(B > 0 && H > 0 && W > 0, "bad loss dims B=%d H=%d W=%d", B, H, W);
    GA_REQUIRE(image && gt && workspace && d_image, "NULL pointer argument");
    if (int rc = ensure_gauss()) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const size_t n = (size_t)B * 3 * H * W;
    Carver c(workspace);
    float *maps = c.take<float>(3 * n);
    (void)c.take<double>(2);
    float *coef = c.take<float>(4);
    { ProfScope _ps("loss_coef_kernel", st); loss_coef_kernel<<<1, 1, 0, st>>>(grad_out, w_l1, w_ssim, (float)(1.0 / (double)n), coef); }
    GA_CHECK_LAUNCH("loss_coef_kernel");
    dim3 grid(cdiv(W, kTX), cdiv(H, kTY), B * 3), block(kTX, kTY);
    { ProfScope _ps("ssim_l1_bwd_kernel", st); ssim_l1_bwd_kernel<<<grid, block, 0, st>>>(H, W, image, gt, maps, maps + n, maps + 2 * n, coef, d_image); }
    GA_CHECK_LAUNCH("ssim_l1_bwd_kernel");
    return GA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Adam (torch.optim.Adam semantics, amsgrad=False, weight_decay=0; model/avatar_model.py:148-155,264-267): one launch per
// parameter buffer.  step is the 1-based step count AFTER increment.
// ---------------------------------------------------------------------------------------------------------------------
namespace ga {
namespace {
// hyper (device, optional): [lr, beta1, beta2, eps, bias_correction1, sqrt(bias_correction2), grad_scale] — read at run time so
// that a captured CUDA graph does not freeze the schedule; skip (device, optional): a non-zero word turns the launch into a
// no-op (the batched rasterizer's overflow flag: a step whose binning buffer overflowed must not be committed).
__global__ void __launch_bounds__(256)
adam_kernel(size_t n, float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v, float lr,
            float beta1, float beta2, float eps, float bc1, float bc2_sqrt, float grad_scale, const float *__restrict__ hyper,
            const int32_t *__restrict__ skip)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (skip && *skip != 0) return;
    if (hyper) { lr = hyper[0]; beta1 = hyper[1]; beta2 = hyper[2]; eps = hyper[3]; bc1 = hyper[4]; bc2_sqrt = hyper[5]; grad_scale = hyper[6]; }
    const float gr = g[i] * grad_scale;
    const float mi = beta1 * m[i] + (1.f - beta1) * gr;       // exp_avg.lerp_(grad, 1 - beta1)
    const float vi = beta2 * v[i] + (1.f - beta2) * gr * gr;  // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] -= (lr / bc1) * (mi / denom);
}
}  // namespace
}  // namespace ga

extern "C" int ga_adam_step(int64_t n, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float lr, float beta1,
                            float beta2, float eps, int64_t step, float grad_scale, const int32_t *skip_flag, void *stream_)
{
    GA_REQUIRE(n >= 0 && step >= 1, "bad adam args n=%lld step=%lld", (long long)n, (long long)step);
    if (n == 0) return GA_OK;
    GA_REQUIRE(param && grad && exp_avg && exp_avg_sq, "NULL pointer argument");
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    { ProfScope _ps("adam_kernel", static_cast<cudaStream_t>(stream_)); adam_kernel<<<cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>((size_t)n, param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps,
                                                                             (float)bc1, (float)sqrt(bc2), grad_scale, nullptr, skip_flag); }
    GA_CHECK_LAUNCH("adam_kernel");
    return GA_OK;
}

extern "C" int ga_adam_step_dev(int64_t n, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, const float *hyper7,
                                const int32_t *skip_flag, void *stream_)
{
    GA_REQUIRE(n >= 0, "bad adam args n=%lld", (long long)n);
    if (n == 0) return GA_OK;
    GA_REQUIRE(param && grad && exp_avg && exp_avg_sq && hyper7, "NULL pointer argument");
    { ProfScope _ps("adam_kernel", static_cast<cudaStream_t>(stream_)); adam_kernel<<<cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>((size_t)n, param, grad, exp_avg, exp_avg_sq, 0.f, 0.f, 0.f, 0.f,
                                                                             1.f, 1.f, 1.f, hyper7, skip_flag); }
    GA_CHECK_LAUNCH("adam_kernel");
    return GA_OK;
}
