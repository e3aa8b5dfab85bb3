// Screen-space mesh renderer: B <= 8 frames of a posed triangle mesh, depth-tested and shaded, drawn with the cameras the Gaussian
// rasterizer takes.  Replaces the reference's pyrender overlay (scripts/render_pred_smpl.py) with exact, deterministic integer
// coverage; see DESIGN.md §4 for the layout and bounds, §2 (PARITY UNPINNED) for what is assumed of pyrender.
//
//   mesh_vertex_kernel        per (vertex, frame): the area-weighted vertex normal (gathered through the vertex -> face CSR, in
//                             CSR order, so no atomics) and the screen position: the Gaussian preprocess's projection (xf_row,
//                             ndc2Pix), snapped to 1/256 pixel, y flipped up so that fixed_raster.cuh's tie rule applies as in
//                             posmap.cu; view-space depth z from the view matrix's third row.
//   mesh_raster_kernel        per (face, frame): a face whose pixel box holds at most kSmallFacePixels centres tests them itself;
//                             a larger one is appended to its frame's list for the tile pass.
//   mesh_raster_tiles_kernel  per (16 x 16 tile, frame): the listed faces (at most F) are set up 256 at a time, those whose box
//                             meets the tile are compacted in shared memory, and every pixel of the tile tests those: a face that
//                             covers the whole frame costs one bounded loop per pixel instead of one unbounded loop in one thread.
//   mesh_shade_kernel         per (pixel, frame): resolves the winner, recomputes its weights and shades it (glTF metallic-roughness
//                             BRDF, one headlight), or writes the background.
//   mesh_unlit_kernel         (ga_mesh_shade_unlit, after ga_mesh_render) per (pixel, frame): the drawn face's weights, recomputed
//                             from its projected corners, interpolate vertex colours or a texture coordinate sampled bilinearly.
//
// Coverage: a pixel is covered when its centre is (pixel (c, r) sits at window position (c, r), as the Gaussians' pixels do).  The
// winner per pixel is the 64-bit atomicMin of (fp32 depth bits << 32) | face: the nearest face, and the lower index at equal
// depth.  The depth is the perspective-correct 1 / sum_i (w_i / z_i) with w_i = E_i / area from the int64 edge functions, in fp64,
// rounded to fp32 once.  No back-face culling.  A face is not drawn when a corner has z <= kZnear (the dataset cameras' near
// plane) or lies outside the +-2^20-pixel guard band (which keeps the edge functions exact in int64): GL would clip such a face
// and draw its visible part.  Every step of the depth path uses explicitly rounded operations (no contraction), mirrored op for
// op by oracle/mesh_oracle.py, so face_id and depth are bit-reproducible and do not depend on the batch a frame is drawn in.
#include "common.cuh"
#include "fixed_raster.cuh"
#include "mesh_project.cuh"

namespace ga {
namespace {

constexpr int kMaxB = 8;
constexpr int kMaxSide = 16384;
using mesh::kCamStride;
constexpr int kSmallFacePixels = 256;
constexpr int kTile = 16;
constexpr unsigned long long kEmpty = ~0ull;
// render_pred_smpl.py's material and light: MetallicRoughnessMaterial(metallicFactor=0.2, roughnessFactor=0.6), intensity 3
constexpr float kMetallic = 0.2f, kRoughness = 0.6f, kLight = 3.f, kPi = 3.14159265358979f;

__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }

__device__ __forceinline__ float dot3(const float a[3], const float b[3]) { return add_(add_(mul_(a[0], b[0]), mul_(a[1], b[1])), mul_(a[2], b[2])); }

// a /= |a|; false (a unchanged) when |a| is 0
__device__ __forceinline__ bool normalize3(float a[3])
{
    const float l2 = dot3(a, a);
    if (!(l2 > 0.f)) return false;
    const float l = __fsqrt_rn(l2);
    a[0] = div_(a[0], l); a[1] = div_(a[1], l); a[2] = div_(a[2], l);
    return true;
}

struct ScreenVert {
    long long x, y;      // 1/256-pixel fixed point, y up
    float z;             // view-space depth
    int ok;              // z > kZnear and inside the guard band
};

struct FaceSetup {
    long long x[3], y[3], area;       // counter-clockwise (y up), area > 0
    float z[3];
    int v[3], f;
    int c0, c1, r0, r1;               // pixel box, inclusive, clipped to the frame
};

__device__ __forceinline__ ScreenVert screen_vert(const float *__restrict__ cam, int H, int W, const float *__restrict__ p)
{
    float pixx, pixy, tvz;
    mesh::project(cam, H, W, p[0], p[1], p[2], pixx, pixy, tvz);
    ScreenVert s;
    s.ok = mesh::drawable(pixx, pixy, tvz);
    s.x = s.ok ? snap_fixed((double)pixx * 256.0) : 0;
    s.y = s.ok ? -snap_fixed((double)pixy * 256.0) : 0;
    s.z = tvz;
    return s;
}

// sv: the screen positions of all vertices, or (sv_local) those of face f's three corners
__device__ __forceinline__ bool setup_face(const ScreenVert *__restrict__ sv, const int *__restrict__ faces, int f, int H, int W, FaceSetup &s,
                                           const ScreenVert *sv_local = nullptr)
{
    s.f = f;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const int vi = faces[3 * (size_t)f + i];
        const ScreenVert q = sv_local ? sv_local[i] : sv[vi];
        if (!q.ok) return false;
        s.v[i] = vi; s.x[i] = q.x; s.y[i] = q.y; s.z[i] = q.z;
    }
    s.area = edge_fn(s.x[0], s.y[0], s.x[1], s.y[1], s.x[2], s.y[2]);
    if (s.area == 0) return false;
    if (s.area < 0) {
        long long tx = s.x[1], ty = s.y[1];
        s.x[1] = s.x[2]; s.y[1] = s.y[2]; s.x[2] = tx; s.y[2] = ty;
        const float tz = s.z[1]; s.z[1] = s.z[2]; s.z[2] = tz;
        const int tv = s.v[1]; s.v[1] = s.v[2]; s.v[2] = tv;
        s.area = -s.area;
    }
    const long long xmin = min(s.x[0], min(s.x[1], s.x[2])), xmax = max(s.x[0], max(s.x[1], s.x[2]));
    const long long ymin = min(s.y[0], min(s.y[1], s.y[2])), ymax = max(s.y[0], max(s.y[1], s.y[2]));
    // centres: column c at x = 256 c, row r at y = -256 r
    s.c0 = (int)max(0LL, (xmin + 255) >> 8);
    s.c1 = (int)min((long long)W - 1, xmax >> 8);
    s.r0 = (int)max(0LL, (-ymax + 255) >> 8);
    s.r1 = (int)min((long long)H - 1, (-ymin) >> 8);
    return s.c0 <= s.c1 && s.r0 <= s.r1;
}

// Whether the face owns the centre of pixel (c, r); e[i] = the edge function opposite corner i (its unnormalised weight).
__device__ __forceinline__ bool covers(const FaceSetup &s, int c, int r, long long e[3])
{
    const long long px = 256LL * c, py = -256LL * r;
    e[0] = edge_fn(s.x[1], s.y[1], s.x[2], s.y[2], px, py);
    e[1] = edge_fn(s.x[2], s.y[2], s.x[0], s.y[0], px, py);
    e[2] = edge_fn(s.x[0], s.y[0], s.x[1], s.y[1], px, py);
    return edge_owns(e[2], s.x[1] - s.x[0], s.y[1] - s.y[0]) && edge_owns(e[0], s.x[2] - s.x[1], s.y[2] - s.y[1]) &&
           edge_owns(e[1], s.x[0] - s.x[2], s.y[0] - s.y[2]);
}

// q[i] = w_i / z_i (fp64); returns sum_i q[i]
__device__ __forceinline__ double inv_depth(const FaceSetup &s, const long long e[3], double q[3])
{
    const double A = __ll2double_rn(s.area);
#pragma unroll
    for (int i = 0; i < 3; ++i) q[i] = __ddiv_rn(__ddiv_rn(__ll2double_rn(e[i]), A), (double)s.z[i]);
    return __dadd_rn(__dadd_rn(q[0], q[1]), q[2]);
}

__device__ __forceinline__ void draw(unsigned long long *__restrict__ key, const FaceSetup &s, const long long e[3])
{
    double q[3];
    const float d = __double2float_rn(__ddiv_rn(1.0, inv_depth(s, e, q)));
    atomicMin(key, ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)s.f);
}

__global__ void __launch_bounds__(128)
mesh_vertex_kernel(int V, int H, int W, const float *__restrict__ verts, const int *__restrict__ faces, const int *__restrict__ adj_off,
                   const int *__restrict__ adj_face, const float *__restrict__ cams, ScreenVert *__restrict__ sv, float *__restrict__ normals)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (v >= V) return;
    const float *X = verts + (size_t)b * V * 3;
    float n[3] = {0.f, 0.f, 0.f};
    for (int k = adj_off[v]; k < adj_off[v + 1]; ++k) {
        const int f = adj_face[k];
        const float *p0 = X + 3 * (size_t)faces[3 * (size_t)f], *p1 = X + 3 * (size_t)faces[3 * (size_t)f + 1],
                    *p2 = X + 3 * (size_t)faces[3 * (size_t)f + 2];
        const float a[3] = {sub_(p1[0], p0[0]), sub_(p1[1], p0[1]), sub_(p1[2], p0[2])};
        const float c[3] = {sub_(p2[0], p0[0]), sub_(p2[1], p0[1]), sub_(p2[2], p0[2])};
        n[0] = add_(n[0], sub_(mul_(a[1], c[2]), mul_(a[2], c[1])));
        n[1] = add_(n[1], sub_(mul_(a[2], c[0]), mul_(a[0], c[2])));
        n[2] = add_(n[2], sub_(mul_(a[0], c[1]), mul_(a[1], c[0])));
    }
    normalize3(n);
    float *no = normals + ((size_t)b * V + v) * 3;
    no[0] = n[0]; no[1] = n[1]; no[2] = n[2];
    sv[(size_t)b * V + v] = screen_vert(cams + (size_t)b * kCamStride, H, W, X + 3 * (size_t)v);
}

__global__ void __launch_bounds__(128)
mesh_raster_kernel(int F, int V, int H, int W, const int *__restrict__ faces, const ScreenVert *__restrict__ sv,
                   unsigned long long *__restrict__ keys, int *__restrict__ big, int *__restrict__ big_count)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (f >= F) return;
    FaceSetup s;
    if (!setup_face(sv + (size_t)b * V, faces, f, H, W, s)) return;
    if ((long long)(s.c1 - s.c0 + 1) * (s.r1 - s.r0 + 1) > kSmallFacePixels) {
        big[(size_t)b * F + atomicAdd(big_count + b, 1)] = f;
        return;
    }
    unsigned long long *kb = keys + (size_t)b * H * W;
    for (int r = s.r0; r <= s.r1; ++r)
        for (int c = s.c0; c <= s.c1; ++c) {
            long long e[3];
            if (covers(s, c, r, e)) draw(kb + (size_t)r * W + c, s, e);
        }
}

__global__ void __launch_bounds__(kTile * kTile)
mesh_raster_tiles_kernel(int F, int V, int H, int W, const int *__restrict__ faces, const ScreenVert *__restrict__ sv,
                         unsigned long long *__restrict__ keys, const int *__restrict__ big, const int *__restrict__ big_count)
{
    __shared__ FaceSetup sf[kTile * kTile];
    __shared__ int s_n;
    const int b = blockIdx.y, tid = threadIdx.x;
    const int tiles_x = (W + kTile - 1) / kTile;
    const int tc0 = (blockIdx.x % tiles_x) * kTile, tr0 = (blockIdx.x / tiles_x) * kTile;
    const int c = tc0 + tid % kTile, r = tr0 + tid / kTile;
    const bool inside = c < W && r < H;
    const int n = big_count[b];
    unsigned long long *key = keys + (size_t)b * H * W + (size_t)r * W + c;
    for (int base = 0; base < n; base += kTile * kTile) {
        __syncthreads();
        if (tid == 0) s_n = 0;
        __syncthreads();
        // the chunk's faces whose box meets this tile, compacted (in any order: the depth test does not depend on it)
        if (base + tid < n) {
            FaceSetup s;
            if (setup_face(sv + (size_t)b * V, faces, big[(size_t)b * F + base + tid], H, W, s) && s.c1 >= tc0 && s.c0 < tc0 + kTile &&
                s.r1 >= tr0 && s.r0 < tr0 + kTile)
                sf[atomicAdd(&s_n, 1)] = s;
        }
        __syncthreads();
        const int m = s_n;
        if (!inside) continue;
        for (int j = 0; j < m; ++j) {
            const FaceSetup &s = sf[j];
            if (c < s.c0 || c > s.c1 || r < s.r0 || r > s.r1) continue;
            long long e[3];
            if (covers(s, c, r, e)) draw(key, s, e);
        }
    }
}

// glTF 2.0 metallic-roughness BRDF (Appendix B) for one directional light l of intensity kLight: Schlick F, height-correlated Smith
// V, GGX D with alpha = roughness^2.  n, l, v unit vectors, n facing the viewer.
__device__ __forceinline__ void shade(const float n[3], const float l[3], const float v[3], const float base[3], float out[3])
{
    const float NdotL = dot3(n, l);
    if (!(NdotL > 0.f)) { out[0] = out[1] = out[2] = 0.f; return; }
    float h[3] = {add_(l[0], v[0]), add_(l[1], v[1]), add_(l[2], v[2])};
    if (!normalize3(h)) { h[0] = l[0]; h[1] = l[1]; h[2] = l[2]; }
    const float NdotV = fmaxf(dot3(n, v), 0.f), NdotH = fmaxf(dot3(n, h), 0.f), VdotH = fmaxf(dot3(v, h), 0.f);
    const float alpha = mul_(kRoughness, kRoughness), a2 = mul_(alpha, alpha), one_a2 = sub_(1.f, a2);
    const float gv = __fsqrt_rn(add_(mul_(mul_(NdotV, NdotV), one_a2), a2));
    const float gl = __fsqrt_rn(add_(mul_(mul_(NdotL, NdotL), one_a2), a2));
    const float vis = div_(0.5f, add_(mul_(NdotL, gv), mul_(NdotV, gl)));
    const float dd = add_(mul_(mul_(NdotH, NdotH), sub_(a2, 1.f)), 1.f);
    const float D = div_(a2, mul_(kPi, mul_(dd, dd)));
    const float t = sub_(1.f, VdotH), t2 = mul_(t, t), t5 = mul_(mul_(t2, t2), t);
    const float one_m = sub_(1.f, kMetallic), li = mul_(kLight, NdotL);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float f0 = add_(mul_(0.04f, one_m), mul_(base[ch], kMetallic));
        const float cdiff = mul_(mul_(base[ch], 0.96f), one_m);
        const float F = add_(f0, mul_(sub_(1.f, f0), t5));
        const float c = mul_(li, add_(div_(mul_(sub_(1.f, F), cdiff), kPi), mul_(mul_(F, vis), D)));
        out[ch] = fminf(fmaxf(c, 0.f), 1.f);
    }
}

__global__ void __launch_bounds__(256)
mesh_shade_kernel(int V, int H, int W, const float *__restrict__ verts, const int *__restrict__ faces, const float *__restrict__ cams,
                  const ScreenVert *__restrict__ sv, const float *__restrict__ normals, const unsigned long long *__restrict__ keys,
                  const float *__restrict__ background, float br, float bg, float bb, int *__restrict__ face_id, float *__restrict__ depth,
                  float *__restrict__ rgb)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    const int n = H * W;
    if (t >= n) return;
    const size_t o = (size_t)b * n + t;
    float *out = rgb + (size_t)b * 3 * n + t;
    const unsigned long long key = keys[o];
    if (key == kEmpty) {
        face_id[o] = -1;
        depth[o] = 0.f;
        const float *bgp = background ? background + (size_t)b * 3 * n + t : nullptr;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) out[(size_t)ch * n] = bgp ? bgp[(size_t)ch * n] : 0.f;
        return;
    }
    const int f = (int)(unsigned int)(key & 0xffffffffu);
    face_id[o] = f;
    depth[o] = __uint_as_float((unsigned int)(key >> 32));

    FaceSetup s;
    setup_face(sv + (size_t)b * V, faces, f, H, W, s);         // succeeds: the face was drawn here
    long long e[3];
    covers(s, t % W, t / W, e);
    double q[3];
    const double sum = inv_depth(s, e, q);
    const float w[3] = {__double2float_rn(__ddiv_rn(q[0], sum)), __double2float_rn(__ddiv_rn(q[1], sum)), __double2float_rn(__ddiv_rn(q[2], sum))};
    const float *X = verts + (size_t)b * V * 3, *N = normals + (size_t)b * V * 3;
    float nrm[3], P[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        nrm[k] = add_(add_(mul_(w[0], N[3 * (size_t)s.v[0] + k]), mul_(w[1], N[3 * (size_t)s.v[1] + k])), mul_(w[2], N[3 * (size_t)s.v[2] + k]));
        P[k] = add_(add_(mul_(w[0], X[3 * (size_t)s.v[0] + k]), mul_(w[1], X[3 * (size_t)s.v[1] + k])), mul_(w[2], X[3 * (size_t)s.v[2] + k]));
    }
    // camera centre C = -R^T t and the headlight l = -(optical axis) = -R^T e_z, from the view matrix (R[r][k] = M[4k + r], t[r] = M[12 + r])
    const float *M = cams + (size_t)b * kCamStride;
    float l[3] = {-M[2], -M[6], -M[10]};
    normalize3(l);
    float v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float Ck = -add_(add_(mul_(M[4 * k], M[12]), mul_(M[4 * k + 1], M[13])), mul_(M[4 * k + 2], M[14]));
        v[k] = sub_(Ck, P[k]);
    }
    if (!normalize3(v)) { v[0] = l[0]; v[1] = l[1]; v[2] = l[2]; }
    if (!normalize3(nrm)) { nrm[0] = l[0]; nrm[1] = l[1]; nrm[2] = l[2]; }
    if (dot3(nrm, v) < 0.f) { nrm[0] = -nrm[0]; nrm[1] = -nrm[1]; nrm[2] = -nrm[2]; }
    const float base[3] = {br, bg, bb};
    float c[3];
    shade(nrm, l, v, base, c);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) out[(size_t)ch * n] = c[ch];
}

// Unlit resolve of a drawn frame: per pixel, the face mesh_shade_kernel resolved there, its perspective-correct weights w_i = q_i / sum
// recomputed in fp64 from the same snapped corners, and either the interpolated vertex colours or a bilinear texture sample at the
// interpolated texture coordinate (glTF's: texel (c, r) centred at ((c + 0.5) / Tw, (r + 0.5) / Th), row 0 first, clamped to the edge).
// Every step is an explicitly rounded fp64 operation, rounded to fp32 once at the end.
__global__ void __launch_bounds__(256)
mesh_unlit_kernel(int V, int F, int H, int W, const float *__restrict__ verts, const int *__restrict__ faces, const float *__restrict__ cams,
                  const int *__restrict__ face_id, const float *__restrict__ colors, const float *__restrict__ uvs, const float *__restrict__ tex,
                  int Th, int Tw, const float *__restrict__ background, float *__restrict__ rgb)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    const int n = H * W;
    if (t >= n) return;
    float *out = rgb + (size_t)b * 3 * n + t;
    const int f = face_id[(size_t)b * n + t];
    const float *X = verts + (size_t)b * V * 3, *cam = cams + (size_t)b * kCamStride;
    FaceSetup s;
    bool drawn = f >= 0 && f < F;
    if (drawn) {
        ScreenVert q[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) q[i] = screen_vert(cam, H, W, X + 3 * (size_t)faces[3 * (size_t)f + i]);
        drawn = setup_face(nullptr, faces, f, H, W, s, q);
    }
    if (!drawn) {
        const float *bgp = background ? background + (size_t)b * 3 * n + t : nullptr;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) out[(size_t)ch * n] = bgp ? bgp[(size_t)ch * n] : 0.f;
        return;
    }
    long long e[3];
    covers(s, t % W, t / W, e);
    double q[3];
    const double sum = inv_depth(s, e, q);
    double w[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) w[i] = __ddiv_rn(q[i], sum);
    const auto lerp3 = [&](const float *a, int stride, int k) {
        return __dadd_rn(__dadd_rn(__dmul_rn(w[0], (double)a[stride * (size_t)s.v[0] + k]), __dmul_rn(w[1], (double)a[stride * (size_t)s.v[1] + k])),
                         __dmul_rn(w[2], (double)a[stride * (size_t)s.v[2] + k]));
    };
    if (colors) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) out[(size_t)ch * n] = __double2float_rn(lerp3(colors, 3, ch));
        return;
    }
    const double x = __dsub_rn(__dmul_rn(lerp3(uvs, 2, 0), (double)Tw), 0.5), y = __dsub_rn(__dmul_rn(lerp3(uvs, 2, 1), (double)Th), 0.5);
    const double x0 = floor(x), y0 = floor(y);
    const double fx = __dsub_rn(x, x0), fy = __dsub_rn(y, y0);
    // NaN or far-off coordinates clamp to the edge too
    const int c0 = x0 >= 0.0 ? (int)fmin(x0, (double)(Tw - 1)) : 0, c1 = x0 + 1.0 >= 0.0 ? (int)fmin(x0 + 1.0, (double)(Tw - 1)) : 0;
    const int r0 = y0 >= 0.0 ? (int)fmin(y0, (double)(Th - 1)) : 0, r1 = y0 + 1.0 >= 0.0 ? (int)fmin(y0 + 1.0, (double)(Th - 1)) : 0;
    const double gx = __dsub_rn(1.0, fx), gy = __dsub_rn(1.0, fy);
    const float *T00 = tex + 3 * ((size_t)r0 * Tw + c0), *T01 = tex + 3 * ((size_t)r0 * Tw + c1);
    const float *T10 = tex + 3 * ((size_t)r1 * Tw + c0), *T11 = tex + 3 * ((size_t)r1 * Tw + c1);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const double top = __dadd_rn(__dmul_rn(gx, (double)T00[ch]), __dmul_rn(fx, (double)T01[ch]));
        const double bot = __dadd_rn(__dmul_rn(gx, (double)T10[ch]), __dmul_rn(fx, (double)T11[ch]));
        out[(size_t)ch * n] = __double2float_rn(__dadd_rn(__dmul_rn(gy, top), __dmul_rn(fy, bot)));
    }
}

struct MeshWs {
    unsigned long long *keys;
    ScreenVert *sv;
    float *normals;
    int *big, *big_count;
    size_t total;
};

MeshWs carve(void *p, int B, int V, int F, int H, int W)
{
    Carver c(p);
    MeshWs w;
    w.keys = c.take<unsigned long long>((size_t)B * H * W);
    w.sv = c.take<ScreenVert>((size_t)B * V);
    w.normals = c.take<float>((size_t)B * V * 3);
    w.big = c.take<int>((size_t)B * F);
    w.big_count = c.take<int>(B);
    w.total = c.used();
    return w;
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" size_t ga_mesh_render_workspace_bytes(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W)
{
    if (B < 0 || V < 0 || F < 0 || H < 0 || W < 0) return 0;
    return carve(nullptr, B, V, F, H, W).total;
}

extern "C" int ga_mesh_render(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, const float *verts, const int32_t *faces,
                              const int32_t *adj_offsets, const int32_t *adj_faces, const float *cams, float base_r, float base_g, float base_b,
                              const float *background, void *workspace, int32_t *face_id, float *depth, float *rgb, void *stream_)
{
    GA_REQUIRE(B >= 0 && B <= kMaxB, "ga_mesh_render: batch %d outside [0, %d]", B, kMaxB);
    GA_REQUIRE(V > 0 && V <= (1 << 24) && F >= 0 && F <= (1 << 24), "ga_mesh_render: bad vertex / face count %d / %d", V, F);
    GA_REQUIRE(H >= 1 && H <= kMaxSide && W >= 1 && W <= kMaxSide, "ga_mesh_render: frame %d x %d outside [1, %d]^2", H, W, kMaxSide);
    if (B == 0) return GA_OK;
    GA_REQUIRE(verts && adj_offsets && cams && workspace && face_id && depth && rgb && (F == 0 || (faces && adj_faces)), "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const MeshWs w = carve(workspace, B, V, F, H, W);
    GA_CHECK_CUDA(cudaMemsetAsync(w.keys, 0xff, sizeof(unsigned long long) * B * H * W, stream));
    GA_CHECK_CUDA(cudaMemsetAsync(w.big_count, 0, sizeof(int) * B, stream));
    { ProfScope _ps("mesh_vertex_kernel", stream);
      mesh_vertex_kernel<<<dim3(cdiv(V, 128), B), 128, 0, stream>>>(V, H, W, verts, faces, adj_offsets, adj_faces, cams, w.sv, w.normals); }
    GA_CHECK_LAUNCH("mesh_vertex_kernel");
    if (F > 0) {
        { ProfScope _ps("mesh_raster_kernel", stream);
          mesh_raster_kernel<<<dim3(cdiv(F, 128), B), 128, 0, stream>>>(F, V, H, W, faces, w.sv, w.keys, w.big, w.big_count); }
        GA_CHECK_LAUNCH("mesh_raster_kernel");
        { ProfScope _ps("mesh_raster_tiles_kernel", stream);
          mesh_raster_tiles_kernel<<<dim3(cdiv(W, kTile) * cdiv(H, kTile), B), kTile * kTile, 0, stream>>>(F, V, H, W, faces, w.sv, w.keys, w.big,
                                                                                                          w.big_count); }
        GA_CHECK_LAUNCH("mesh_raster_tiles_kernel");
    }
    { ProfScope _ps("mesh_shade_kernel", stream);
      mesh_shade_kernel<<<dim3(cdiv((long long)H * W, 256), B), 256, 0, stream>>>(V, H, W, verts, faces, cams, w.sv, w.normals, w.keys, background,
                                                                                  base_r, base_g, base_b, face_id, depth, rgb); }
    GA_CHECK_LAUNCH("mesh_shade_kernel");
    return GA_OK;
}

extern "C" int ga_mesh_shade_unlit(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, const float *verts, const int32_t *faces,
                                   const float *cams, const int32_t *face_id, const float *colors, const float *uvs, const float *texture,
                                   int32_t Th, int32_t Tw, const float *background, float *rgb, void *stream_)
{
    GA_REQUIRE(B >= 1 && B <= kMaxB, "ga_mesh_shade_unlit: batch %d outside [1, %d]", B, kMaxB);
    GA_REQUIRE(V > 0 && V <= (1 << 24) && F >= 0 && F <= (1 << 24), "ga_mesh_shade_unlit: bad vertex / face count %d / %d", V, F);
    GA_REQUIRE(H >= 1 && H <= kMaxSide && W >= 1 && W <= kMaxSide, "ga_mesh_shade_unlit: frame %d x %d outside [1, %d]^2", H, W, kMaxSide);
    GA_REQUIRE((colors != nullptr) != (uvs != nullptr || texture != nullptr),
               "ga_mesh_shade_unlit: give vertex colours or texture coordinates and a texture, not both");
    GA_REQUIRE(colors || (uvs && texture && Th >= 1 && Th <= kMaxSide && Tw >= 1 && Tw <= kMaxSide),
               "ga_mesh_shade_unlit: texture %d x %d outside [1, %d]^2 or a NULL texture / texture coordinates", Th, Tw, kMaxSide);
    GA_REQUIRE(verts && cams && face_id && rgb && (F == 0 || faces), "ga_mesh_shade_unlit: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("mesh_unlit_kernel", stream);
      mesh_unlit_kernel<<<dim3(cdiv((long long)H * W, 256), B), 256, 0, stream>>>(V, F, H, W, verts, faces, cams, face_id, colors, uvs, texture,
                                                                                  Th, Tw, background, rgb); }
    GA_CHECK_LAUNCH("mesh_unlit_kernel");
    return GA_OK;
}
