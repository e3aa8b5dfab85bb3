// Device math shared by the SMPL kernels (smpl.cu: joint transforms; posmap.cu: posed mesh vertices).
#pragma once
#include <cuda_runtime.h>

namespace ga {

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

}  // namespace ga
