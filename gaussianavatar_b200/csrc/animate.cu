// Animation player kernels: sampling a motion clip at fractional key times, and packing rendered frames into interleaved bytes.
//
//   motion_sample_kernel  per (output frame, joint): keys i = floor(tau), i + 1 of the clip as unit quaternions (the second
//                         negated when their dot product is negative), slerp at f = tau - i (normalised lerp above a dot of
//                         1 - 1e-12), the root pre-multiplied by the alignment rotation, back to axis-angle with w >= 0 (angle in
//                         [0, pi]); the root thread also writes R_a lerp(t_i, t_i+1, f) + c.  Everything in fp64, rounded to fp32 once.
//   frame_pack_kernel     per (pixel, frame): save_image's byte quantisation q(x) = uint8(clamp(fp32(fp32(x 255) + 0.5), 0, 255))
//                         (NaN -> 0) of the rendered colour, interleaved HWC; with 4 channels the colour is first un-composited from
//                         the constant background (the rasterizer wrote C + T bg) and the fourth byte is q(1 - T).  Every rounding
//                         is explicit (__fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn), so nvcc cannot contract them into an FMA and
//                         oracle/animate_oracle.py restates the bytes exactly.
#include "common.cuh"

namespace ga {
namespace {

constexpr int kPackMaxB = 8;
constexpr int kPackMaxSide = 16384;
constexpr double kNlerpDot = 1.0 - 1e-12;

struct Quat { double w, x, y, z; };

__device__ __forceinline__ Quat quat_from_aa(double vx, double vy, double vz)
{
    const double th = sqrt(vx * vx + vy * vy + vz * vz);
    const double h = 0.5 * th;
    const double s = th > 1e-8 ? sin(h) / th : 0.5 - th * th / 48.0;     // sin(th/2)/th, its series below 1e-8
    return Quat{cos(h), s * vx, s * vy, s * vz};
}

// Shepperd's method: the largest of 4w^2, 4x^2, 4y^2, 4z^2 picks the branch, so no square root of a small difference is taken.
__device__ __forceinline__ Quat quat_from_mat(const double *R)
{
    const double tr = R[0] + R[4] + R[8];
    Quat q;
    if (tr >= R[0] && tr >= R[4] && tr >= R[8]) {
        const double s = 2.0 * sqrt(1.0 + tr);
        q = Quat{0.25 * s, (R[7] - R[5]) / s, (R[2] - R[6]) / s, (R[3] - R[1]) / s};
    } else if (R[0] >= R[4] && R[0] >= R[8]) {
        const double s = 2.0 * sqrt(1.0 + R[0] - R[4] - R[8]);
        q = Quat{(R[7] - R[5]) / s, 0.25 * s, (R[1] + R[3]) / s, (R[2] + R[6]) / s};
    } else if (R[4] >= R[8]) {
        const double s = 2.0 * sqrt(1.0 + R[4] - R[0] - R[8]);
        q = Quat{(R[2] - R[6]) / s, (R[1] + R[3]) / s, 0.25 * s, (R[5] + R[7]) / s};
    } else {
        const double s = 2.0 * sqrt(1.0 + R[8] - R[0] - R[4]);
        q = Quat{(R[3] - R[1]) / s, (R[2] + R[6]) / s, (R[5] + R[7]) / s, 0.25 * s};
    }
    const double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    return Quat{q.w / n, q.x / n, q.y / n, q.z / n};
}

__device__ __forceinline__ Quat quat_mul(const Quat &a, const Quat &b)
{
    return Quat{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
                a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}

__device__ __forceinline__ Quat slerp(Quat a, Quat b, double f)
{
    double d = a.w * b.w + a.x * b.x + a.y * b.y + a.z * b.z;
    if (d < 0.0) { b = Quat{-b.w, -b.x, -b.y, -b.z}; d = -d; }
    double ca, cb;
    if (d > kNlerpDot) {
        ca = 1.0 - f; cb = f;
    } else {
        const double om = acos(d), so = sin(om);
        ca = sin((1.0 - f) * om) / so; cb = sin(f * om) / so;
    }
    Quat q{ca * a.w + cb * b.w, ca * a.x + cb * b.x, ca * a.y + cb * b.y, ca * a.z + cb * b.z};
    const double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    return Quat{q.w / n, q.x / n, q.y / n, q.z / n};
}

__global__ void motion_sample_kernel(int T, int J, int n, const float *__restrict__ key_pose, const float *__restrict__ key_trans,
                                     const double *__restrict__ times, const double *__restrict__ align, float *__restrict__ pose_out,
                                     float *__restrict__ trans_out)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * J) return;
    const int k = t / J, j = t - k * J;
    const double tau = fmin(fmax(times[k], 0.0), (double)(T - 1));        // fmax(NaN, 0) = 0
    const int i0 = min((int)floor(tau), T - 1);
    const int i1 = min(i0 + 1, T - 1);
    const double f = tau - (double)i0;
    const float *p0 = key_pose + (size_t)i0 * J * 3 + j * 3, *p1 = key_pose + (size_t)i1 * J * 3 + j * 3;
    Quat q = slerp(quat_from_aa(p0[0], p0[1], p0[2]), quat_from_aa(p1[0], p1[1], p1[2]), f);
    double R[9];
    if (j == 0) {
#pragma unroll
        for (int e = 0; e < 9; ++e) R[e] = align[e];
        q = quat_mul(quat_from_mat(R), q);
    }
    if (q.w < 0.0) q = Quat{-q.w, -q.x, -q.y, -q.z};
    const double s = sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    const double g = s > 0.0 ? 2.0 * atan2(s, q.w) / s : 0.0;                // angle / |v|
    float *po = pose_out + (size_t)k * J * 3 + j * 3;
    po[0] = (float)(g * q.x);
    po[1] = (float)(g * q.y);
    po[2] = (float)(g * q.z);
    if (j == 0) {
        const float *a = key_trans + (size_t)i0 * 3, *b = key_trans + (size_t)i1 * 3;
        double v[3];
#pragma unroll
        for (int e = 0; e < 3; ++e) v[e] = (double)a[e] + f * ((double)b[e] - (double)a[e]);
#pragma unroll
        for (int r = 0; r < 3; ++r)
            trans_out[(size_t)k * 3 + r] = (float)(R[3 * r] * v[0] + R[3 * r + 1] * v[1] + R[3 * r + 2] * v[2] + align[9 + r]);
    }
}

__device__ __forceinline__ uint8_t quant8(float x)
{
    const float y = __fadd_rn(__fmul_rn(x, 255.f), 0.5f);
    if (!(y >= 0.f)) return 0;                 // negative or NaN
    return (uint8_t)(y < 255.f ? y : 255.f);   // truncation, as torch's .to(uint8)
}

template <int C>
__global__ void frame_pack_kernel(long long HW, const float *__restrict__ image, const float *__restrict__ final_T,
                                  const float *__restrict__ bg, uint8_t *__restrict__ out)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const int b = blockIdx.y;
    const float *im = image + (size_t)b * 3 * HW + p;
    const float x0 = im[0], x1 = im[HW], x2 = im[2 * HW];
    uint8_t *o = out + ((size_t)b * HW + p) * C;
    if (C == 3) {
        o[0] = quant8(x0); o[1] = quant8(x1); o[2] = quant8(x2);
    } else {
        const float Tr = final_T[(size_t)b * HW + p];
        const float a = __fsub_rn(1.f, Tr);
        const uint8_t A = quant8(a);
        uchar4 v = make_uchar4(0, 0, 0, 0);
        if (A != 0) {
            v.x = quant8(__fdiv_rn(__fsub_rn(x0, __fmul_rn(Tr, bg[0])), a));
            v.y = quant8(__fdiv_rn(__fsub_rn(x1, __fmul_rn(Tr, bg[1])), a));
            v.z = quant8(__fdiv_rn(__fsub_rn(x2, __fmul_rn(Tr, bg[2])), a));
            v.w = A;
        }
        *reinterpret_cast<uchar4 *>(o) = v;
    }
}

__global__ void matte_pack_kernel(long long n, const float *__restrict__ mattes, uint8_t *__restrict__ out)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = quant8(mattes[i]);
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_motion_sample(int32_t T, int32_t J, const float *key_pose, const float *key_trans, int32_t n, const double *times,
                                const double *align, float *pose_out, float *trans_out, void *stream_)
{
    GA_REQUIRE(T >= 1, "ga_motion_sample: clip of %d keys (need >= 1)", T);
    GA_REQUIRE(J == 24 || J == 55, "ga_motion_sample: %d joints (24 for SMPL, 55 for SMPL-X)", J);
    GA_REQUIRE(n >= 1 && (long long)n * J <= 0x7fffffffll, "ga_motion_sample: %d output frames", n);
    GA_REQUIRE(key_pose && key_trans && times && align && pose_out && trans_out, "ga_motion_sample: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const long long threads = (long long)n * J;
    { ProfScope _ps("motion_sample_kernel", stream);
      motion_sample_kernel<<<cdiv(threads, 128), 128, 0, stream>>>(T, J, n, key_pose, key_trans, times, align, pose_out, trans_out); }
    GA_CHECK_LAUNCH("motion_sample_kernel");
    return GA_OK;
}

extern "C" int ga_frame_pack(int32_t B, int32_t H, int32_t W, int32_t channels, const float *image, const float *final_T, const float *bg,
                             uint8_t *out, void *stream_)
{
    GA_REQUIRE(B >= 1 && B <= kPackMaxB, "ga_frame_pack: batch %d outside [1, %d]", B, kPackMaxB);
    GA_REQUIRE(H >= 1 && H <= kPackMaxSide && W >= 1 && W <= kPackMaxSide, "ga_frame_pack: frame %d x %d outside [1, %d]^2", H, W,
               kPackMaxSide);
    GA_REQUIRE(channels == 3 || channels == 4, "ga_frame_pack: %d channels (3: RGB, 4: RGBA)", channels);
    GA_REQUIRE(image && out && (channels == 3 || (final_T && bg)), "ga_frame_pack: NULL pointer argument");
    GA_REQUIRE(channels == 3 || reinterpret_cast<uintptr_t>(out) % 4 == 0, "ga_frame_pack: RGBA output must be 4-byte aligned");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const long long HW = (long long)H * W;
    const dim3 grid(cdiv(HW, 256), B);
    { ProfScope _ps("frame_pack_kernel", stream);
      if (channels == 3) frame_pack_kernel<3><<<grid, 256, 0, stream>>>(HW, image, final_T, bg, out);
      else frame_pack_kernel<4><<<grid, 256, 0, stream>>>(HW, image, final_T, bg, out); }
    GA_CHECK_LAUNCH("frame_pack_kernel");
    return GA_OK;
}

extern "C" int ga_matte_pack(int64_t n, const float *mattes, uint8_t *out, void *stream_)
{
    GA_REQUIRE(n >= 1, "ga_matte_pack: %lld values", (long long)n);
    GA_REQUIRE(mattes && out, "ga_matte_pack: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("matte_pack_kernel", stream);
      matte_pack_kernel<<<min(cdiv(n, 256), 1 << 20), 256, 0, stream>>>(n, mattes, out); }
    GA_CHECK_LAUNCH("matte_pack_kernel");
    return GA_OK;
}
