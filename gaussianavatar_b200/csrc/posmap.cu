// Stage-2 input position maps on the device: posed SMPL mesh vertices, the UV-space coverage layout, and the per-frame fill.
//
// Replaces the reference's offline pipeline scripts/gen_pose_map_our_smpl.py (smplx forward -> OBJ per frame -> PosRender in a GLUT
// window, shaders pos_uv.vs / pos_uv.fs).  The rasterization happens in UV space (gl_Position = 2 (uv - 0.5)), so which face
// covers which texel, and with which barycentric weights, depends only on the UV template and the map size: ga_posmap_layout
// computes it once, and a frame costs ga_smpl_vertices (pose blend shapes + LBS) and ga_posmap_fill (a gather of three vertices
// per texel).
//
// Coverage rules of ga_posmap_layout (the GL spec leaves them open; see DESIGN.md, PARITY UNPINNED):
//   - window coordinates (u S, v S), snapped to 1/256 texel: X = rint(u * 256 S) (round half to even, exact in fp64);
//   - a texel is covered when its centre is: column c, output row r samples X = 256 c + 128, Y = 256 (S - r) - 128 (the
//     reference's get_color flips the rows, so row 0 is the top, v near 1);
//   - edge functions in int64; a point on an edge belongs to the face only if the edge, walked counter-clockwise (y up), goes
//     down (dy < 0) or, when horizontal, to the left (dy == 0, dx < 0).  Two faces that share an edge traverse it in opposite
//     directions, so each centre on it is covered exactly once; a face of zero area covers nothing;
//   - no culling; all depths are 0 and the depth test is GL_LESS, so where faces overlap the lowest face index wins;
//   - a face with a non-finite corner or a corner coordinate of magnitude above 4096 covers nothing (keeps the int64 edge
//     functions exact);
//   - barycentric weights from the snapped coordinates: w_i = E_i / area in fp64, rounded to fp32.
#include "common.cuh"
#include "smpl_math.cuh"

namespace ga {
namespace {

constexpr int kJoints = 24;
constexpr int kPoseFeat = 9 * (kJoints - 1);     // 207 pose blend-shape coefficients
constexpr int kMaxB = 8;
constexpr int kVertsPerCta = 32;
constexpr int kCols = 3 * kVertsPerCta;          // posedirs columns per CTA
constexpr int kRowGroups = 4;                    // posedirs rows split over this many thread groups
constexpr int kVertThreads = kCols * kRowGroups;
constexpr int kNoFace = 0x7f7f7f7f;                // face_id before the raster pass: every byte 0x7f (one memset)
constexpr int kMaxS = 512;

__constant__ int c_parents_v[kJoints] = {-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21};

// Posed vertices of B <= 8 frames.  Every CTA first forms the B frames' pose features and joint transforms A (joint j's global
// transform is the product of its ancestors' local transforms, one lane per joint, so no chain walk), then streams its 96 columns
// of posedirs [207, 3V] ONCE for all B frames (four row groups, reduced in shared memory), then skins its 32 vertices.
__global__ void __launch_bounds__(kVertThreads)
smpl_vertices_kernel(int B, int V, const float *__restrict__ pose /*[B,72]*/, const float *__restrict__ transl /*[B,3]*/,
                     const float *__restrict__ J /*[24,3]*/, const float *__restrict__ v_shaped /*[V,3]*/,
                     const float *__restrict__ posedirs /*[207,3V]*/, const float *__restrict__ weights /*[V,24]*/,
                     float *__restrict__ verts /*[B,V,3]*/)
{
    __shared__ float sL[kMaxB][kJoints][12], sA[kMaxB][kJoints][12];
    __shared__ float sFeat[kMaxB][kPoseFeat];
    __shared__ float sPart[kRowGroups][kMaxB][kCols];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (warp < B && lane < kJoints) {
        const int b = warp, j = lane;
        const float r[3] = {pose[b * 72 + j * 3], pose[b * 72 + j * 3 + 1], pose[b * 72 + j * 3 + 2]};
        float R[9], th;
        rodrigues(r, R, &th);
        const int p = c_parents_v[j];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            sL[b][j][k * 4 + 0] = R[k * 3 + 0]; sL[b][j][k * 4 + 1] = R[k * 3 + 1]; sL[b][j][k * 4 + 2] = R[k * 3 + 2];
            sL[b][j][k * 4 + 3] = (p < 0) ? J[j * 3 + k] : (J[j * 3 + k] - J[p * 3 + k]);
        }
        if (j > 0) {
#pragma unroll
            for (int k = 0; k < 9; ++k) sFeat[b][(j - 1) * 9 + k] = R[k] - ((k % 4 == 0) ? 1.f : 0.f);
        }
    }
    __syncthreads();
    if (warp < B && lane < kJoints) {
        const int b = warp, j = lane;
        float G[12], T[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) G[k] = sL[b][j][k];
        for (int p = c_parents_v[j]; p >= 0; p = c_parents_v[p]) {
            aff_mul(sL[b][p], G, T);
#pragma unroll
            for (int k = 0; k < 12; ++k) G[k] = T[k];
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            sA[b][j][r * 4 + 0] = G[r * 4 + 0]; sA[b][j][r * 4 + 1] = G[r * 4 + 1]; sA[b][j][r * 4 + 2] = G[r * 4 + 2];
            sA[b][j][r * 4 + 3] = G[r * 4 + 3] - (G[r * 4 + 0] * J[j * 3] + G[r * 4 + 1] * J[j * 3 + 1] + G[r * 4 + 2] * J[j * 3 + 2]);
        }
    }
    __syncthreads();

    // pose blend shapes: column k of posedirs, rows rg, rg + 4, ...; one accumulator per frame
    const int col = tid % kCols, rg = tid / kCols;
    const long long ncol = 3LL * V;
    const long long k = (long long)blockIdx.x * kCols + col;
    float acc[kMaxB];
#pragma unroll
    for (int b = 0; b < kMaxB; ++b) acc[b] = 0.f;
    if (k < ncol) {
#pragma unroll 4
        for (int r = rg; r < kPoseFeat; r += kRowGroups) {
            const float pd = __ldg(posedirs + (long long)r * ncol + k);
#pragma unroll
            for (int b = 0; b < kMaxB; ++b)
                if (b < B) acc[b] = fmaf(sFeat[b][r], pd, acc[b]);
        }
    }
#pragma unroll
    for (int b = 0; b < kMaxB; ++b)
        if (b < B) sPart[rg][b][col] = acc[b];
    __syncthreads();

    // skinning: T = sum_j w_vj A_j, x = T [v_posed; 1] + transl
    for (int i = tid; i < kVertsPerCta * B; i += kVertThreads) {
        const int vl = i % kVertsPerCta, b = i / kVertsPerCta;
        const int v = blockIdx.x * kVertsPerCta + vl;
        if (v >= V) continue;
        float x[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float off = 0.f;
#pragma unroll
            for (int g = 0; g < kRowGroups; ++g) off += sPart[g][b][vl * 3 + c];
            x[c] = v_shaped[(size_t)v * 3 + c] + off;
        }
        float T[12];
#pragma unroll
        for (int q = 0; q < 12; ++q) T[q] = 0.f;
        const float *w = weights + (size_t)v * kJoints;
        for (int j = 0; j < kJoints; ++j) {
            const float wj = w[j];
#pragma unroll
            for (int q = 0; q < 12; ++q) T[q] = fmaf(wj, sA[b][j][q], T[q]);
        }
        float *o = verts + ((size_t)b * V + v) * 3;
#pragma unroll
        for (int r = 0; r < 3; ++r)
            o[r] = T[r * 4 + 0] * x[0] + T[r * 4 + 1] * x[1] + T[r * 4 + 2] * x[2] + T[r * 4 + 3] + transl[b * 3 + r];
    }
}

struct Snapped { long long x[3], y[3]; bool ok; };

__device__ __forceinline__ Snapped snap_face(const float *__restrict__ uv, int f, int S)
{
    Snapped s;
    s.ok = true;
    const double scale = 256.0 * S;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float u = uv[(size_t)f * 6 + i * 2], v = uv[(size_t)f * 6 + i * 2 + 1];
        if (!(fabsf(u) <= 4096.f) || !(fabsf(v) <= 4096.f)) s.ok = false;     // also false for NaN
        s.x[i] = s.ok ? __double2ll_rn((double)u * scale) : 0;
        s.y[i] = s.ok ? __double2ll_rn((double)v * scale) : 0;
    }
    return s;
}

// edge function of (a -> b) at p: > 0 when p is to the left (y up)
__device__ __forceinline__ long long edge_fn(long long ax, long long ay, long long bx, long long by, long long px, long long py)
{
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}

__device__ __forceinline__ bool edge_owns(long long e, long long dx, long long dy)
{
    return e > 0 || (e == 0 && (dy < 0 || (dy == 0 && dx < 0)));
}

// One thread per face: walk the texel centres of its bounding box and keep the lowest covering face index per texel.
__global__ void __launch_bounds__(128)
posmap_raster_kernel(int F, int S, const float *__restrict__ uv, int *__restrict__ face_id)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    Snapped s = snap_face(uv, f, S);
    if (!s.ok) return;
    long long area = edge_fn(s.x[0], s.y[0], s.x[1], s.y[1], s.x[2], s.y[2]);
    if (area == 0) return;
    if (area < 0) {            // counter-clockwise from here on
        long long tx = s.x[1], ty = s.y[1];
        s.x[1] = s.x[2]; s.y[1] = s.y[2]; s.x[2] = tx; s.y[2] = ty;
    }
    const long long xmin = min(s.x[0], min(s.x[1], s.x[2])), xmax = max(s.x[0], max(s.x[1], s.x[2]));
    const long long ymin = min(s.y[0], min(s.y[1], s.y[2])), ymax = max(s.y[0], max(s.y[1], s.y[2]));
    // centres 256 i + 128 inside [min, max]
    const long long c0 = max(0LL, (xmin - 128 + 255) >> 8), c1 = min((long long)S - 1, (xmax - 128) >> 8);
    const long long k0 = max(0LL, (ymin - 128 + 255) >> 8), k1 = min((long long)S - 1, (ymax - 128) >> 8);
    for (long long k = k0; k <= k1; ++k) {
        const long long py = 256 * k + 128;
        for (long long c = c0; c <= c1; ++c) {
            const long long px = 256 * c + 128;
            bool in = true;
#pragma unroll
            for (int e = 0; e < 3; ++e) {
                const int a = e, b = (e + 1) % 3;
                in = in && edge_owns(edge_fn(s.x[a], s.y[a], s.x[b], s.y[b], px, py), s.x[b] - s.x[a], s.y[b] - s.y[a]);
            }
            if (in) atomicMin(face_id + (S - 1 - k) * S + c, f);       // window row k is output row S-1-k
        }
    }
}

// One thread per texel: -1 / zero weights where nothing covers it, else the covering face's barycentric weights.
__global__ void __launch_bounds__(256)
posmap_resolve_kernel(int F, int S, const float *__restrict__ uv, int *__restrict__ face_id, float *__restrict__ bary)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= S * S) return;
    const int f = face_id[t];
    float w[3] = {0.f, 0.f, 0.f};
    if (f < 0 || f >= F) {         // kNoFace: nothing covers the texel
        face_id[t] = -1;
    } else {
        const Snapped s = snap_face(uv, f, S);
        const int r = t / S, c = t % S;
        const long long px = 256LL * c + 128, py = 256LL * (S - r) - 128;
        const double area = (double)edge_fn(s.x[0], s.y[0], s.x[1], s.y[1], s.x[2], s.y[2]);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const int a = (i + 1) % 3, b = (i + 2) % 3;
            w[i] = (float)((double)edge_fn(s.x[a], s.y[a], s.x[b], s.y[b], px, py) / area);
        }
    }
    bary[(size_t)t * 3 + 0] = w[0]; bary[(size_t)t * 3 + 1] = w[1]; bary[(size_t)t * 3 + 2] = w[2];
}

// out[b, :, r, c] = sum_i w_i x_b[faces[f, i]] (fp32, i in order), 0 where face_id is -1.  One thread per (texel, frame).
__global__ void __launch_bounds__(256)
posmap_fill_kernel(int S, int V, const float *__restrict__ verts, const int *__restrict__ faces, const int *__restrict__ face_id,
                   const float *__restrict__ bary, float *__restrict__ out)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    const int n = S * S;
    if (t >= n) return;
    const int f = face_id[t];
    float o[3] = {0.f, 0.f, 0.f};
    if (f >= 0) {
        const float *xb = verts + (size_t)b * V * 3;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float w = bary[(size_t)t * 3 + i];
            const float *p = xb + (size_t)faces[(size_t)f * 3 + i] * 3;
            o[0] = fmaf(w, p[0], o[0]); o[1] = fmaf(w, p[1], o[1]); o[2] = fmaf(w, p[2], o[2]);
        }
    }
    float *ob = out + (size_t)b * 3 * n;
    ob[t] = o[0]; ob[n + t] = o[1]; ob[2 * n + t] = o[2];
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_smpl_vertices(int32_t B, int32_t V, const float *pose, const float *transl, const float *rest_joints,
                                const float *v_shaped, const float *posedirs, const float *weights, float *verts, void *stream_)
{
    GA_REQUIRE(B >= 0 && B <= kMaxB, "ga_smpl_vertices: batch %d outside [0, %d]", B, kMaxB);
    GA_REQUIRE(V > 0 && V <= (1 << 24), "ga_smpl_vertices: bad vertex count %d", V);
    if (B == 0) return GA_OK;
    GA_REQUIRE(pose && transl && rest_joints && v_shaped && posedirs && weights && verts, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("smpl_vertices_kernel", stream);
      smpl_vertices_kernel<<<cdiv(V, kVertsPerCta), kVertThreads, 0, stream>>>(B, V, pose, transl, rest_joints, v_shaped, posedirs,
               weights, verts); }
    GA_CHECK_LAUNCH("smpl_vertices_kernel");
    return GA_OK;
}

extern "C" int ga_posmap_layout(int32_t F, int32_t S, const float *uv_corners, int32_t *face_id, float *bary, void *stream_)
{
    GA_REQUIRE(F >= 0 && F < kNoFace, "ga_posmap_layout: bad face count %d", F);
    GA_REQUIRE(S >= 1 && S <= kMaxS, "ga_posmap_layout: map size %d outside [1, %d]", S, kMaxS);
    GA_REQUIRE(face_id && bary && (F == 0 || uv_corners), "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    GA_CHECK_CUDA(cudaMemsetAsync(face_id, 0x7f, sizeof(int32_t) * S * S, stream));      // kNoFace > any face index
    if (F > 0) {
        { ProfScope _ps("posmap_raster_kernel", stream); posmap_raster_kernel<<<cdiv(F, 128), 128, 0, stream>>>(F, S, uv_corners, face_id); }
        GA_CHECK_LAUNCH("posmap_raster_kernel");
    }
    { ProfScope _ps("posmap_resolve_kernel", stream); posmap_resolve_kernel<<<cdiv(S * S, 256), 256, 0, stream>>>(F, S, uv_corners, face_id, bary); }
    GA_CHECK_LAUNCH("posmap_resolve_kernel");
    return GA_OK;
}

extern "C" int ga_posmap_fill(int32_t B, int32_t S, int32_t V, const float *verts, const int32_t *faces, const int32_t *face_id,
                              const float *bary, float *out, void *stream_)
{
    GA_REQUIRE(B >= 0 && B <= 65535, "ga_posmap_fill: bad batch %d", B);
    GA_REQUIRE(S >= 1 && S <= kMaxS && V > 0, "ga_posmap_fill: bad map size %d / vertex count %d", S, V);
    if (B == 0) return GA_OK;
    GA_REQUIRE(verts && faces && face_id && bary && out, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("posmap_fill_kernel", stream);
      posmap_fill_kernel<<<dim3(cdiv(S * S, 256), B), 256, 0, stream>>>(S, V, verts, faces, face_id, bary, out); }
    GA_CHECK_LAUNCH("posmap_fill_kernel");
    return GA_OK;
}
