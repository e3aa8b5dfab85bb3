// Body-model device math shared by smpl.cu (joint transforms, forward and backward) and posmap.cu (posed mesh vertices, forward and
// backward): the SMPL / SMPL-X kinematic trees and body traits, the per-joint steps from axis-angle to rest-relative transform, and
// Rodrigues with its backward.  posmap.cu's forward and backward vertex kernels form their joint transforms through these routines, so
// the backward rebuilds exactly what the forward computed.
#pragma once
#include <cuda_runtime.h>

namespace ga {

constexpr int kSmplJoints = 24, kSmplxJoints = 55;

namespace {     // per translation unit (the library is built without -rdc)
__constant__ int c_parents_smpl[kSmplJoints] = {-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21};
// SMPL-X (global, 21 body, jaw, left / right eye, 2 x 15 finger joints): kintree_table[0] of SMPLX_*.npz (the asset loader checks
// the model file against this table)
__constant__ int c_parents_smplx[kSmplxJoints] = {-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15,
                                                  20, 25, 26, 20, 28, 29, 20, 31, 32, 20, 34, 35, 20, 37, 38, 21, 40, 41, 21, 43, 44, 21,
                                                  46, 47, 21, 49, 50, 21, 52, 53};
}  // namespace

// A body of kJ joints: the first kTrained read from `pose` [B, 3 kTrained], the rest from `rest_pose` [B, 3 (kJ - kTrained)]; kFeat
// pose blend-shape coefficients (R_j - I of every joint but the root); parent(j), -1 for the root and below j otherwise.
template <int kJ> struct Body;
template <> struct Body<kSmplJoints> {
    static constexpr int kTrained = 24, kFeat = 9 * (kSmplJoints - 1);
    static __device__ __forceinline__ int parent(int j) { return c_parents_smpl[j]; }
};
template <> struct Body<kSmplxJoints> {
    static constexpr int kTrained = 22, kFeat = 9 * (kSmplxJoints - 1);
    static __device__ __forceinline__ int parent(int j) { return c_parents_smplx[j]; }
};

// 3x4 affine helpers (row-major, implicit last row 0 0 0 1)
__device__ __forceinline__ void aff_mul(const float *A, const float *B, float *C)  // C = A * B
{
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float t = A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c] + A[r * 4 + 2] * B[2 * 4 + c];
            if (c == 3) t += A[r * 4 + 3];
            C[r * 4 + c] = t;
        }
    }
}

// Rodrigues with the reference's shifted norm: theta = |r + 1e-8| (submodules/smplx/lbs.py:317)
__device__ __forceinline__ void rodrigues(const float r[3], float R[9], float *theta_out)
{
    const float nx = r[0] + 1e-8f, ny = r[1] + 1e-8f, nz = r[2] + 1e-8f;
    const float theta = sqrtf(nx * nx + ny * ny + nz * nz);
    const float dx = r[0] / theta, dy = r[1] / theta, dz = r[2] / theta;
    float s, c;
    sincosf(theta, &s, &c);
    const float K[9] = {0.f, -dz, dy, dz, 0.f, -dx, -dy, dx, 0.f};
    float K2[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) K2[i * 3 + j] = K[i * 3] * K[j] + K[i * 3 + 1] * K[3 + j] + K[i * 3 + 2] * K[6 + j];
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.f : 0.f) + s * K[i] + (1.f - c) * K2[i];
    *theta_out = theta;
}

// Backward of rodrigues(): R = I + s K + (1 - c) K^2 with K the cross matrix of d = r / theta, theta = |r + 1e-8|.
// smpl_bwd_kernel keeps its own inline copy, whose results differ from this one's in the last bits (DESIGN.md §7).
__device__ __forceinline__ void rodrigues_bwd(const float r[3], const float gR[9], float gr[3])
{
    const float n[3] = {r[0] + 1e-8f, r[1] + 1e-8f, r[2] + 1e-8f};
    const float theta = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    const float dx = r[0] / theta, dy = r[1] / theta, dz = r[2] / theta;
    float s, c;
    sincosf(theta, &s, &c);
    const float K[9] = {0.f, -dz, dy, dz, 0.f, -dx, -dy, dx, 0.f};
    float K2[9], gK[9];
    float gs = 0.f, g1c = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) K2[i * 3 + j] = K[i * 3] * K[j] + K[i * 3 + 1] * K[3 + j] + K[i * 3 + 2] * K[6 + j];
#pragma unroll
    for (int i = 0; i < 9; ++i) { gs = fmaf(gR[i], K[i], gs); g1c = fmaf(gR[i], K2[i], g1c); }
    // d(K^2) = dK K + K dK: gK = s gR + (1 - c) (gR K^T + K^T gR)
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float t = 0.f;
#pragma unroll
            for (int k = 0; k < 3; ++k) t += gR[i * 3 + k] * K[j * 3 + k] + K[k * 3 + i] * gR[k * 3 + j];
            gK[i * 3 + j] = s * gR[i * 3 + j] + (1.f - c) * t;
        }
    const float gd[3] = {gK[7] - gK[5], gK[2] - gK[6], gK[3] - gK[1]};
    float gth = gs * c + g1c * s - (gd[0] * r[0] + gd[1] * r[1] + gd[2] * r[2]) / (theta * theta);
#pragma unroll
    for (int k = 0; k < 3; ++k) gr[k] = gd[k] / theta + gth * n[k] / theta;
}

// axis-angle of joint j of frame b (rest_pose is not read for SMPL, whose joints all come from pose)
template <int kJ>
__device__ __forceinline__ void joint_axis_angle(const float *__restrict__ pose, const float *__restrict__ rest_pose, int b, int j, float r[3])
{
    constexpr int kT = Body<kJ>::kTrained;
    if (kT == kJ || j < kT) {
        r[0] = pose[(size_t)b * (kT * 3) + j * 3]; r[1] = pose[(size_t)b * (kT * 3) + j * 3 + 1]; r[2] = pose[(size_t)b * (kT * 3) + j * 3 + 2];
    } else {
        const int k = j - kT;
        r[0] = rest_pose[(size_t)b * ((kJ - kT) * 3) + k * 3]; r[1] = rest_pose[(size_t)b * ((kJ - kT) * 3) + k * 3 + 1];
        r[2] = rest_pose[(size_t)b * ((kJ - kT) * 3) + k * 3 + 2];
    }
}

// local transform of joint j (rotation | offset to its parent) from its rotation R
template <int kJ>
__device__ __forceinline__ void local_transform(const float R[9], const float *__restrict__ J, int j, float *L)
{
    const int p = Body<kJ>::parent(j);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        L[k * 4 + 0] = R[k * 3 + 0]; L[k * 4 + 1] = R[k * 3 + 1]; L[k * 4 + 2] = R[k * 3 + 2];
        L[k * 4 + 3] = (p < 0) ? J[j * 3 + k] : (J[j * 3 + k] - J[p * 3 + k]);
    }
}

// global transform of joint j: the product of its ancestors' local transforms, root first
template <int kJ>
__device__ __forceinline__ void chain_product(const float (*L)[12], int j, float G[12])
{
    float T[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) G[k] = L[j][k];
    for (int p = Body<kJ>::parent(j); p >= 0; p = Body<kJ>::parent(p)) {
        aff_mul(L[p], G, T);
#pragma unroll
        for (int k = 0; k < 12; ++k) G[k] = T[k];
    }
}

// A = G - pad(G_R J_j): joint j's transform relative to the rest pose (lbs.py:402-403)
__device__ __forceinline__ void rest_relative(const float *G, const float *__restrict__ J, int j, float A[12])
{
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        A[r * 4 + 0] = G[r * 4 + 0]; A[r * 4 + 1] = G[r * 4 + 1]; A[r * 4 + 2] = G[r * 4 + 2];
        A[r * 4 + 3] = G[r * 4 + 3] - (G[r * 4 + 0] * J[j * 3] + G[r * 4 + 1] * J[j * 3 + 1] + G[r * 4 + 2] * J[j * 3 + 2]);
    }
}

}  // namespace ga
