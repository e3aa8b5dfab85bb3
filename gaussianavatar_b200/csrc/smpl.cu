// SMPL / SMPL-X joint transforms -> canonical-to-live matrices, forward + backward, one CTA per pose.
//
// Replaces `smpl_model.forward(...).A` followed by `torch.matmul(live_smpl.A, self.inv_mats)`
// (/root/reference model/avatar_model.py:291-296), i.e. submodules/smplx/lbs.py:152-252 reduced to what feeds A:
// Rodrigues with the shifted norm (:299-333), the 23-step kinematic chain (:349-405, a Python loop of ~150 tiny kernel
// launches in the reference), `A = G - pad(G J)` (:402-403), `A[:, :, :3, 3] += transl` (body_models.py:380-383).
// The rest joints J depend only on the (fixed) betas and are precomputed once on the host side.
//
// Both kernels are templates over the body model:
//   SMPL    24 joints, all trainable (pose [B,72]); one warp per pose.
//   SMPL-X  55 joints (global, 21 body, jaw, left / right eye, 15 + 15 finger joints), the first 22 trainable (pose [B,66]), the
//           other 33 read from rest_pose [B,99] (jaw, eyes, hands: data, never differentiated); a 64-thread CTA per pose.
//           The chain is 54 dependent 3x4 products walked in index order, a few microseconds with no bandwidth at stake.
#include "common.cuh"
#include "smpl_math.cuh"

namespace ga {
namespace {

__constant__ int c_parents[24] = {-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21};
// SMPL-X kintree_table[0] (the asset loader checks the model file against this table)
__constant__ int c_parents_x[55] = {-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15, 20, 25,
                                    26, 20, 28, 29, 20, 31, 32, 20, 34, 35, 20, 37, 38, 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50,
                                    21, 52, 53};

// kJ joints, the first kTrain of them from `pose` [B, 3 kTrain], the rest from `rest` [B, 3 (kJ - kTrain)]; kThreads per CTA
template <int kJ> struct Body;
template <> struct Body<24> { static constexpr int kTrain = 24, kThreads = 32; };
template <> struct Body<55> { static constexpr int kTrain = 22, kThreads = 64; };

template <int kJ> __device__ __forceinline__ int parent_of(int j) { return kJ == 24 ? c_parents[j] : c_parents_x[j]; }

template <int kThreads> __device__ __forceinline__ void cta_sync()
{
    if constexpr (kThreads == 32) __syncwarp();
    else __syncthreads();
}

// axis-angle of joint j of pose b
template <int kJ> __device__ __forceinline__ void load_axis_angle(const float *__restrict__ pose, const float *__restrict__ rest, int b, int j, float r[3])
{
    constexpr int kT = Body<kJ>::kTrain;
    if (kT == kJ || j < kT) {
        r[0] = pose[(size_t)b * (kT * 3) + j * 3]; r[1] = pose[(size_t)b * (kT * 3) + j * 3 + 1]; r[2] = pose[(size_t)b * (kT * 3) + j * 3 + 2];
    } else {
        const int k = j - kT;
        r[0] = rest[(size_t)b * ((kJ - kT) * 3) + k * 3]; r[1] = rest[(size_t)b * ((kJ - kT) * 3) + k * 3 + 1];
        r[2] = rest[(size_t)b * ((kJ - kT) * 3) + k * 3 + 2];
    }
}

// One block (kThreads) per pose.  Thread j < kJ owns joint j for the per-joint steps; the chain itself is walked
// in index order through shared memory (children always have a larger index than their parent).
template <int kJ>
__global__ void __launch_bounds__(Body<kJ>::kThreads)
smpl_fwd_kernel(int B, const float *__restrict__ pose, const float *__restrict__ transl, const float *__restrict__ J,
                const float *__restrict__ inv_cano /*[kJ,4,4]*/, float *__restrict__ C /*[B,kJ,12]*/,
                float *__restrict__ G_out /*[B,kJ,12] saved for backward*/, const float *__restrict__ rest /*[B,99] (SMPL-X)*/)
{
    constexpr int kThreads = Body<kJ>::kThreads;
    __shared__ float sL[kJ][12], sG[kJ][12];
    const int b = blockIdx.x, j = threadIdx.x;
    if (b >= B) return;
    if (j < kJ) {
        float r[3];
        load_axis_angle<kJ>(pose, rest, b, j, r);
        float R[9], th;
        rodrigues(r, R, &th);
        const int p = parent_of<kJ>(j);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            sL[j][k * 4 + 0] = R[k * 3 + 0]; sL[j][k * 4 + 1] = R[k * 3 + 1]; sL[j][k * 4 + 2] = R[k * 3 + 2];
            sL[j][k * 4 + 3] = (p < 0) ? J[j * 3 + k] : (J[j * 3 + k] - J[p * 3 + k]);
        }
        if (j == 0) {
#pragma unroll
            for (int k = 0; k < 12; ++k) sG[0][k] = sL[0][k];
        }
    }
    cta_sync<kThreads>();
    // kJ - 1 dependent 3x4 products: thread 0 walks the chain (latency ~ a few microseconds, B poses run in parallel CTAs)
    for (int i = 1; i < kJ; ++i) {
        if (j == 0) aff_mul(sG[parent_of<kJ>(i)], sL[i], sG[i]);
        cta_sync<kThreads>();
    }
    if (j < kJ) {
        float A[12];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            A[r * 4 + 0] = sG[j][r * 4 + 0]; A[r * 4 + 1] = sG[j][r * 4 + 1]; A[r * 4 + 2] = sG[j][r * 4 + 2];
            A[r * 4 + 3] = sG[j][r * 4 + 3] - (sG[j][r * 4 + 0] * J[j * 3] + sG[j][r * 4 + 1] * J[j * 3 + 1] + sG[j][r * 4 + 2] * J[j * 3 + 2]) +
                           transl[(size_t)b * 3 + r];
        }
        // cano2live = A * inv(A_cano)  (both affine)
        const float *Ic = inv_cano + j * 16;
        float *Cj = C + ((size_t)b * kJ + j) * 12;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float t = A[r * 4 + 0] * Ic[0 * 4 + c] + A[r * 4 + 1] * Ic[1 * 4 + c] + A[r * 4 + 2] * Ic[2 * 4 + c] + A[r * 4 + 3] * Ic[3 * 4 + c];
                Cj[r * 4 + c] = t;
            }
        float *Gj = G_out + ((size_t)b * kJ + j) * 12;
#pragma unroll
        for (int k = 0; k < 12; ++k) Gj[k] = sG[j][k];
    }
}

// d_pose [B, 3 kTrain] only: the rest_pose joints of SMPL-X are data.
template <int kJ>
__global__ void __launch_bounds__(Body<kJ>::kThreads)
smpl_bwd_kernel(int B, const float *__restrict__ pose, const float *__restrict__ J, const float *__restrict__ inv_cano,
                const float *__restrict__ G_saved, const float *__restrict__ dC /*[B,kJ,12]*/,
                float *__restrict__ d_pose /*[B,3 kTrain]*/, float *__restrict__ d_transl /*[B,3]*/, const float *__restrict__ rest)
{
    constexpr int kThreads = Body<kJ>::kThreads, kT = Body<kJ>::kTrain;
    __shared__ float sL[kJ][12], sG[kJ][12], sdG[kJ][12], sdL[kJ][9];
    const int b = blockIdx.x, j = threadIdx.x;
    if (b >= B) return;
    float r[3] = {0.f, 0.f, 0.f}, R[9], theta = 1.f;
    if (j < kJ) {
        load_axis_angle<kJ>(pose, rest, b, j, r);
        rodrigues(r, R, &theta);
        const int p = parent_of<kJ>(j);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            sL[j][k * 4 + 0] = R[k * 3 + 0]; sL[j][k * 4 + 1] = R[k * 3 + 1]; sL[j][k * 4 + 2] = R[k * 3 + 2];
            sL[j][k * 4 + 3] = (p < 0) ? J[j * 3 + k] : (J[j * 3 + k] - J[p * 3 + k]);
        }
        const float *Gj = G_saved + ((size_t)b * kJ + j) * 12;
#pragma unroll
        for (int k = 0; k < 12; ++k) sG[j][k] = Gj[k];
        // dA[:3,:4] = dC[:3,:4] * inv_cano^T   (C = A * Ic, rows of A are 4-vectors)
        const float *Ic = inv_cano + j * 16;
        const float *dCj = dC + ((size_t)b * kJ + j) * 12;
        float dA[12];
#pragma unroll
        for (int rr = 0; rr < 3; ++rr)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                dA[rr * 4 + k] = dCj[rr * 4 + 0] * Ic[k * 4 + 0] + dCj[rr * 4 + 1] * Ic[k * 4 + 1] + dCj[rr * 4 + 2] * Ic[k * 4 + 2] + dCj[rr * 4 + 3] * Ic[k * 4 + 3];
        // A_R = G_R ; A_t = G_t - G_R J + transl
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) {
            sdG[j][rr * 4 + 0] = dA[rr * 4 + 0] - dA[rr * 4 + 3] * J[j * 3 + 0];
            sdG[j][rr * 4 + 1] = dA[rr * 4 + 1] - dA[rr * 4 + 3] * J[j * 3 + 1];
            sdG[j][rr * 4 + 2] = dA[rr * 4 + 2] - dA[rr * 4 + 3] * J[j * 3 + 2];
            sdG[j][rr * 4 + 3] = dA[rr * 4 + 3];
        }
    }
    cta_sync<kThreads>();
    // d transl = sum_j dA_t
    if (j == 0) {
        float t0 = 0.f, t1 = 0.f, t2 = 0.f;
        for (int k = 0; k < kJ; ++k) { t0 += sdG[k][3]; t1 += sdG[k][7]; t2 += sdG[k][11]; }
        d_transl[(size_t)b * 3 + 0] = t0; d_transl[(size_t)b * 3 + 1] = t1; d_transl[(size_t)b * 3 + 2] = t2;
    }
    cta_sync<kThreads>();
    // reverse chain: G_i = G_p * L_i
    if (j == 0) {
        for (int i = kJ - 1; i >= 1; --i) {
            const int p = parent_of<kJ>(i);
            const float *Gp = sG[p], *Li = sL[i], *dGi = sdG[i];
            // dL_R = Gp_R^T dGi_R ; (dL_t not needed: J is constant)
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    sdL[i][a * 3 + c] = Gp[0 * 4 + a] * dGi[0 * 4 + c] + Gp[1 * 4 + a] * dGi[1 * 4 + c] + Gp[2 * 4 + a] * dGi[2 * 4 + c];
            // dGp_R += dGi_R L_R^T + dGi_t (x) L_t ; dGp_t += dGi_t
#pragma unroll
            for (int a = 0; a < 3; ++a) {
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    sdG[p][a * 4 + c] += dGi[a * 4 + 0] * Li[c * 4 + 0] + dGi[a * 4 + 1] * Li[c * 4 + 1] + dGi[a * 4 + 2] * Li[c * 4 + 2] + dGi[a * 4 + 3] * Li[c * 4 + 3];
                sdG[p][a * 4 + 3] += dGi[a * 4 + 3];
            }
        }
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int c = 0; c < 3; ++c) sdL[0][a * 3 + c] = sdG[0][a * 4 + c];
    }
    cta_sync<kThreads>();
    if (j < kT) {
        // Rodrigues backward.  R = I + s K + (1-c) K^2, K = skew(d), d = r/theta, theta = |r + 1e-8|
        const float *dR = sdL[j];
        const float dx = r[0] / theta, dy = r[1] / theta, dz = r[2] / theta;
        float s, c;
        sincosf(theta, &s, &c);
        const float K[9] = {0.f, -dz, dy, dz, 0.f, -dx, -dy, dx, 0.f};
        float K2[9];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int k = 0; k < 3; ++k) K2[i * 3 + k] = K[i * 3] * K[k] + K[i * 3 + 1] * K[3 + k] + K[i * 3 + 2] * K[6 + k];
        float ds = 0.f, dcm = 0.f;
#pragma unroll
        for (int i = 0; i < 9; ++i) { ds += dR[i] * K[i]; dcm += dR[i] * K2[i]; }
        // dK = s dR + (1-c) (dR K^T + K^T dR)
        float dK[9];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) {
                float t = 0.f;
#pragma unroll
                for (int k = 0; k < 3; ++k) t += dR[a * 3 + k] * K[cc * 3 + k] + K[k * 3 + a] * dR[k * 3 + cc];
                dK[a * 3 + cc] = s * dR[a * 3 + cc] + (1.f - c) * t;
            }
        float dd[3] = {dK[7] - dK[5], dK[2] - dK[6], dK[3] - dK[1]};
        float dtheta = ds * c + dcm * s;   // d/dtheta [s] = c ; d/dtheta [(1-c)] = s
        float dr[3] = {dd[0] / theta, dd[1] / theta, dd[2] / theta};
        dtheta += -(dd[0] * r[0] + dd[1] * r[1] + dd[2] * r[2]) / (theta * theta);
        const float nx = r[0] + 1e-8f, ny = r[1] + 1e-8f, nz = r[2] + 1e-8f;
        dr[0] += dtheta * nx / theta; dr[1] += dtheta * ny / theta; dr[2] += dtheta * nz / theta;
        d_pose[(size_t)b * (kT * 3) + j * 3 + 0] = dr[0];
        d_pose[(size_t)b * (kT * 3) + j * 3 + 1] = dr[1];
        d_pose[(size_t)b * (kT * 3) + j * 3 + 2] = dr[2];
    }
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_smpl_forward(int32_t B, const float *pose, const float *transl, const float *rest_joints,
                               const float *inv_cano, float *cano2live, float *saved_G, void *stream_)
{
    GA_REQUIRE(B >= 0, "bad batch %d", B);
    if (B == 0) return GA_OK;
    GA_REQUIRE(pose && transl && rest_joints && inv_cano && cano2live && saved_G, "NULL pointer argument");
    { ProfScope _ps("smpl_fwd_kernel", static_cast<cudaStream_t>(stream_)); smpl_fwd_kernel<24><<<B, 32, 0, static_cast<cudaStream_t>(stream_)>>>(B, pose, transl, rest_joints, inv_cano, cano2live, saved_G, nullptr); }
    GA_CHECK_LAUNCH("smpl_fwd_kernel");
    return GA_OK;
}

extern "C" int ga_smpl_backward(int32_t B, const float *pose, const float *rest_joints, const float *inv_cano,
                                const float *saved_G, const float *d_cano2live, float *d_pose, float *d_transl, void *stream_)
{
    GA_REQUIRE(B >= 0, "bad batch %d", B);
    if (B == 0) return GA_OK;
    GA_REQUIRE(pose && rest_joints && inv_cano && saved_G && d_cano2live && d_pose && d_transl, "NULL pointer argument");
    { ProfScope _ps("smpl_bwd_kernel", static_cast<cudaStream_t>(stream_)); smpl_bwd_kernel<24><<<B, 32, 0, static_cast<cudaStream_t>(stream_)>>>(B, pose, rest_joints, inv_cano, saved_G, d_cano2live, d_pose, d_transl, nullptr); }
    GA_CHECK_LAUNCH("smpl_bwd_kernel");
    return GA_OK;
}

extern "C" int ga_smplx_forward(int32_t B, const float *pose, const float *rest_pose, const float *transl, const float *rest_joints,
                                const float *inv_cano, float *cano2live, float *saved_G, void *stream_)
{
    GA_REQUIRE(B >= 0, "bad batch %d", B);
    if (B == 0) return GA_OK;
    GA_REQUIRE(pose && rest_pose && transl && rest_joints && inv_cano && cano2live && saved_G, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("smplx_fwd_kernel", stream); smpl_fwd_kernel<55><<<B, Body<55>::kThreads, 0, stream>>>(B, pose, transl, rest_joints, inv_cano, cano2live, saved_G, rest_pose); }
    GA_CHECK_LAUNCH("smplx_fwd_kernel");
    return GA_OK;
}

extern "C" int ga_smplx_backward(int32_t B, const float *pose, const float *rest_pose, const float *rest_joints, const float *inv_cano,
                                 const float *saved_G, const float *d_cano2live, float *d_pose, float *d_transl, void *stream_)
{
    GA_REQUIRE(B >= 0, "bad batch %d", B);
    if (B == 0) return GA_OK;
    GA_REQUIRE(pose && rest_pose && rest_joints && inv_cano && saved_G && d_cano2live && d_pose && d_transl, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("smplx_bwd_kernel", stream); smpl_bwd_kernel<55><<<B, Body<55>::kThreads, 0, stream>>>(B, pose, rest_joints, inv_cano, saved_G, d_cano2live, d_pose, d_transl, rest_pose); }
    GA_CHECK_LAUNCH("smplx_bwd_kernel");
    return GA_OK;
}
