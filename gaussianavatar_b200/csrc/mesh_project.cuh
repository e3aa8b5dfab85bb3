// Screen projection shared by the mesh renderer (mesh_render.cu) and the soft silhouette (silhouette.cu): the Gaussian preprocess's
// projection and pixel convention, and the rule for which vertices a face may be drawn from.
#pragma once

namespace ga {
namespace mesh {

constexpr int kCamStride = 40;                   // the ga_rasterb_* camera block: view 0..15, proj 16..31, tan(fov/2) 32..33
constexpr float kZnear = 0.01f;                  // the dataset cameras' near plane
constexpr float kGuard = 1048576.f;              // 2^20 pixels: |fixed-point coordinate| <= 2^28, edge products < 2^59

// the op order of raster.cu's xf_row (row r of the transposed 4x4 M applied to (x, y, z, 1))
__device__ __forceinline__ float xf_row(const float *__restrict__ M, int r, float x, float y, float z)
{
    float t = __fmul_rn(M[r], x);
    t = __fmaf_rn(M[4 + r], y, t);
    t = __fmaf_rn(M[8 + r], z, t);
    return __fadd_rn(t, M[12 + r]);
}

// Window position (pixx, pixy) of world point (x, y, z) in an H x W frame (pixel (c, r) centred at (c, r), y down) and its
// view-space depth z: full_proj_transform, divide by w, ndc2Pix, rounded to fp32 once.
__device__ __forceinline__ void project(const float *__restrict__ cam, int H, int W, float x, float y, float z, float &pixx, float &pixy,
                                        float &vz)
{
    const float *view = cam, *proj = cam + 16;
    vz = xf_row(view, 2, x, y, z);
    const float hx = xf_row(proj, 0, x, y, z), hy = xf_row(proj, 1, x, y, z), hw = xf_row(proj, 3, x, y, z);
    const float p_w = __fdiv_rn(1.f, __fadd_rn(hw, 0.0000001f));
    const float ndc_x = __fmul_rn(hx, p_w), ndc_y = __fmul_rn(hy, p_w);
    pixx = (float)__dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)ndc_x, 1.0), (double)W), -1.0), 0.5);
    pixy = (float)__dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)ndc_y, 1.0), (double)H), -1.0), 0.5);
}

// Whether a face may use this vertex: in front of the near plane and inside the guard band (false for NaN).  A face with a corner
// that fails is not drawn.
__device__ __forceinline__ bool drawable(float pixx, float pixy, float vz)
{
    return vz > kZnear && fabsf(pixx) <= kGuard && fabsf(pixy) <= kGuard;
}

}  // namespace mesh
}  // namespace ga
