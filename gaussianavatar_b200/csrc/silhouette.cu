// Soft silhouette of a posed triangle mesh and its gradient with respect to the vertices: B <= 8 frames, the cameras the Gaussian
// rasterizer takes.  The function (DESIGN.md §2, PARITY UNPINNED; in the spirit of SoftRas / pytorch3d's SoftSilhouetteShader):
//
//   x_f(p) = +d_f(p)^2 / sigma inside face f's projected triangle, -d_f(p)^2 / sigma outside, d_f = Euclidean distance from the pixel
//            centre p (pixel (c, r) at (c, r)) to the triangle; D_f = sigmoid(x_f), and D_f = 0 outside beyond
//            d_f^2 > sigma ln(1/eps - 1), eps = 1e-4 (the truncation radius);
//   S(p)   = 1 - prod_f (1 - D_f(p)),  loss_b = mean_p (S - M)^2 with M = (mask byte >= 128).
//
// Vertices are projected as mesh_render.cu projects them (mesh_project.cuh), but not snapped; a face with a corner behind the near
// plane or outside the guard band, or with zero projected area, contributes nothing.  No culling.
//
// (1 - S) is kept as its logarithm L(p) = -sum_f softplus(x_f), since log(1 - sigmoid(x)) = -softplus(x): S = -expm1(L) and
// dS/dx_f = D_f exp(L) exactly, so no saturated factor (1 - D_f = 0 in fp32) is ever divided out.  The gradient of d_f^2 is that
// of the nearest edge segment a -> b: with t the clamped projection parameter and q = a + t (b - a), d(d^2)/da = -2 (p - q)(1 - t)
// and d(d^2)/db = -2 (p - q) t, which covers both the edge interior (0 < t < 1) and the vertex (t = 0 or 1) pieces.
//
//   sil_setup_kernel      per (face, frame): projects the three corners, writes the face's corners and its pixel box grown by the
//                         truncation radius (empty for a face that contributes nothing).
//   sil_tile_kernel       per (16 x 16 tile, frame): every face whose box meets the tile, 256 at a time, compacted in face order
//                         (ballots, no atomics); each pixel accumulates L over them in ascending face order.  Writes S and one
//                         partial sum of (S - M)^2 per tile (forward), or G = w_b dloss_b/dS exp(L) per pixel (backward).
//   sil_loss_kernel       per frame: the tile partials summed in a fixed order (fp64), divided by H W.
//   sil_face_grad_kernel  per (face, frame), one warp: the face's six screen-coordinate gradients, sum over its box's pixels of
//                         G D_f dx_f/dcoords, lanes striding the box, then a fixed shuffle tree.  A face covering the whole frame is
//                         one warp's loop over H W pixels.
//   sil_vertex_grad_kernel per (vertex, frame): the faces' corner gradients gathered through the vertex -> face CSR in its order, then
//                         the projection's Jacobian.
//
// Every buffer is sized by the shapes (no capacity, no overflow path), there are no floating-point atomics and no host read-back:
// the outputs are bit-reproducible and a frame's do not depend on the batch it is in.
#include "common.cuh"
#include "mesh_project.cuh"

namespace ga {
namespace {

constexpr int kMaxB = 8;
constexpr int kMaxSide = 16384;
constexpr int kTile = 16;
constexpr int kThreads = kTile * kTile;
constexpr float kLnInvEps = 9.21024036697585f;       // ln(1 / 1e-4 - 1)
using mesh::kCamStride;

struct FaceXY {
    float x[3], y[3];
};

__device__ __forceinline__ float softplus(float x) { return x > 0.f ? x + log1pf(expf(-x)) : log1pf(expf(x)); }
__device__ __forceinline__ float sigmoid(float x)
{
    if (x >= 0.f) return 1.f / (1.f + expf(-x));
    const float e = expf(x);
    return e / (1.f + e);
}

struct Near {
    float x;         // signed d^2 / sigma
    float t;         // projection parameter on the nearest edge
    float dx, dy;    // p - q, q the nearest point of the triangle's boundary
    int edge;        // nearest edge k: corner k -> corner (k + 1) % 3
    bool inside;
};

// Face f at pixel centre (px, py): false where D_f is truncated to 0.  The per-edge geometry is evaluated in fp64 from the fp32
// corners: a corner may lie anywhere in the 2^20-pixel guard band, and near an edge of length l, w - t e cancels to an error of
// ~1e-7 l in fp32, which moved d^2 by up to ~0.3 for a corner 10^6 pixels away (tests/test_silhouette_kernels_gpu.py, long-edge
// tier).  d^2, t and p - q are rounded to fp32 once; softplus, sigmoid and the sums stay in fp32.
__device__ __forceinline__ bool eval_face(const FaceXY &f, float px, float py, float inv_sigma, float trunc_d2, Near &n)
{
    double best = INFINITY, bt = 0.0, bdx = 0.0, bdy = 0.0;
    bool pos = true, neg = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int k1 = k == 2 ? 0 : k + 1;
        const double ax = f.x[k], ay = f.y[k];
        const double ex = (double)f.x[k1] - ax, ey = (double)f.y[k1] - ay;
        const double wx = (double)px - ax, wy = (double)py - ay;
        const double cr = ex * wy - ey * wx;
        pos = pos && cr >= 0.0;
        neg = neg && cr <= 0.0;
        const double t = fmin(fmax((wx * ex + wy * ey) / (ex * ex + ey * ey), 0.0), 1.0);
        const double dx = wx - t * ex, dy = wy - t * ey;
        const double d2 = dx * dx + dy * dy;
        if (d2 < best) { best = d2; bt = t; bdx = dx; bdy = dy; n.edge = k; }
    }
    n.inside = pos || neg;
    if (!n.inside && best > (double)trunc_d2) return false;
    const float b32 = (float)best;
    n.x = (n.inside ? b32 : -b32) * inv_sigma;
    n.t = (float)bt;
    n.dx = (float)bdx;
    n.dy = (float)bdy;
    return true;
}

__global__ void __launch_bounds__(128)
sil_setup_kernel(int F, int V, int H, int W, float trunc_d2, const float *__restrict__ verts, const int *__restrict__ faces,
                 const float *__restrict__ cams, int4 *__restrict__ boxes, FaceXY *__restrict__ xy)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (f >= F) return;
    const float *X = verts + (size_t)b * V * 3, *cam = cams + (size_t)b * kCamStride;
    FaceXY s;
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float *p = X + 3 * (size_t)faces[3 * (size_t)f + i];
        float z;
        mesh::project(cam, H, W, p[0], p[1], p[2], s.x[i], s.y[i], z);
        ok = ok && mesh::drawable(s.x[i], s.y[i], z);
    }
    const float area = (s.x[1] - s.x[0]) * (s.y[2] - s.y[0]) - (s.y[1] - s.y[0]) * (s.x[2] - s.x[0]);
    ok = ok && area != 0.f && isfinite(area);
    int4 box = make_int4(1, 0, 1, 0);                    // c0, c1, r0, r1: empty
    if (ok) {
        const float r = sqrtf(trunc_d2);
        const float x0 = fminf(s.x[0], fminf(s.x[1], s.x[2])) - r, x1 = fmaxf(s.x[0], fmaxf(s.x[1], s.x[2])) + r;
        const float y0 = fminf(s.y[0], fminf(s.y[1], s.y[2])) - r, y1 = fmaxf(s.y[0], fmaxf(s.y[1], s.y[2])) + r;
        box = make_int4(max(0, (int)ceilf(x0)), min(W - 1, (int)floorf(x1)), max(0, (int)ceilf(y0)), min(H - 1, (int)floorf(y1)));
        if (box.x > box.y || box.z > box.w) box = make_int4(1, 0, 1, 0);
    }
    boxes[(size_t)b * F + f] = box;
    xy[(size_t)b * F + f] = s;
}

// Fixed-order sum over the block (every thread passes a value; thread 0 gets the result).
__device__ __forceinline__ float block_sum(float v, float *s_warp)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_warp[warp] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x == 0)
        for (int w = 0; w < kThreads / 32; ++w) t += s_warp[w];
    return t;
}

__global__ void __launch_bounds__(kThreads)
sil_tile_kernel(int F, int H, int W, float inv_sigma, float trunc_d2, const int4 *__restrict__ boxes, const FaceXY *__restrict__ xy,
                const unsigned char *__restrict__ mask, const float *__restrict__ w, float *__restrict__ sil, float *__restrict__ partial,
                float *__restrict__ grad_pix)
{
    __shared__ FaceXY s_xy[kThreads];
    __shared__ int4 s_box[kThreads];
    __shared__ int s_count[kThreads / 32];
    __shared__ float s_red[kThreads / 32];
    const int b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tiles_x = (W + kTile - 1) / kTile;
    const int tc0 = (blockIdx.x % tiles_x) * kTile, tr0 = (blockIdx.x / tiles_x) * kTile;
    const int c = tc0 + tid % kTile, r = tr0 + tid / kTile;
    const bool in_frame = c < W && r < H;
    const float px = (float)c, py = (float)r;
    float L = 0.f;
    for (int base = 0; base < F; base += kThreads) {
        const int f = base + tid;
        int4 box = make_int4(1, 0, 1, 0);
        if (f < F) box = boxes[(size_t)b * F + f];
        const bool hit = box.x <= box.y && box.y >= tc0 && box.x < tc0 + kTile && box.w >= tr0 && box.z < tr0 + kTile;
        const unsigned ballot = __ballot_sync(0xffffffffu, hit);
        __syncthreads();                                  // the previous chunk's faces are no longer read
        if (lane == 0) s_count[warp] = __popc(ballot);
        __syncthreads();
        int pos = __popc(ballot & ((1u << lane) - 1u)), m = 0;
        for (int k = 0; k < kThreads / 32; ++k) {
            if (k < warp) pos += s_count[k];
            m += s_count[k];
        }
        if (hit) { s_xy[pos] = xy[(size_t)b * F + f]; s_box[pos] = box; }
        __syncthreads();
        if (!in_frame) continue;
        for (int j = 0; j < m; ++j) {
            const int4 bx = s_box[j];
            if (c < bx.x || c > bx.y || r < bx.z || r > bx.w) continue;
            Near n;
            if (eval_face(s_xy[j], px, py, inv_sigma, trunc_d2, n)) L -= softplus(n.x);
        }
    }
    const size_t o = (size_t)b * H * W + (size_t)r * W + c;
    const float S = -expm1f(L);
    const float M = (in_frame && mask) ? (mask[o] >= 128 ? 1.f : 0.f) : 0.f;
    if (grad_pix) {
        if (in_frame) grad_pix[o] = w[b] * (2.f * (S - M) / ((float)H * (float)W)) * expf(L);
        return;
    }
    if (in_frame) sil[o] = S;
    if (partial) {
        const float e = in_frame ? (S - M) * (S - M) : 0.f;
        const float t = block_sum(e, s_red);
        if (tid == 0) partial[(size_t)b * gridDim.x + blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kThreads)
sil_loss_kernel(int tiles, int H, int W, const float *__restrict__ partial, float *__restrict__ loss)
{
    __shared__ double s[kThreads];
    const int b = blockIdx.x;
    double t = 0.0;
    for (int i = threadIdx.x; i < tiles; i += kThreads) t += (double)partial[(size_t)b * tiles + i];
    s[threadIdx.x] = t;
    __syncthreads();
    for (int h = kThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) loss[b] = (float)(s[0] / ((double)H * (double)W));
}

__global__ void __launch_bounds__(256)
sil_face_grad_kernel(int F, int H, int W, float inv_sigma, float trunc_d2, const int4 *__restrict__ boxes, const FaceXY *__restrict__ xy,
                     const float *__restrict__ grad_pix, float *__restrict__ fgrad)
{
    const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), b = blockIdx.y, lane = threadIdx.x & 31;
    if (f >= F) return;
    const int4 box = boxes[(size_t)b * F + f];
    const FaceXY s = xy[(size_t)b * F + f];
    float g[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};             // d/d(x0, y0, x1, y1, x2, y2)
    if (box.x <= box.y) {
        const int bw = box.y - box.x + 1;
        const long long n = (long long)bw * (box.w - box.z + 1);
        const float *G = grad_pix + (size_t)b * H * W;
        for (long long k = lane; k < n; k += 32) {
            const int r = box.z + (int)(k / bw), c = box.x + (int)(k % bw);
            Near q;
            if (!eval_face(s, (float)c, (float)r, inv_sigma, trunc_d2, q)) continue;
            // G D_f dx/d(d^2) times d(d^2)/da = -2 (p - q)(1 - t), d(d^2)/db = -2 (p - q) t
            const float coef = -2.f * G[(size_t)r * W + c] * sigmoid(q.x) * (q.inside ? inv_sigma : -inv_sigma);
            const int a = q.edge, e = a == 2 ? 0 : a + 1;
            const float ca = coef * (1.f - q.t), cb = coef * q.t;
            g[2 * a] += ca * q.dx; g[2 * a + 1] += ca * q.dy;
            g[2 * e] += cb * q.dx; g[2 * e + 1] += cb * q.dy;
        }
    }
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) g[i] += __shfl_xor_sync(0xffffffffu, g[i], o);
    if (lane == 0) {
        float *out = fgrad + ((size_t)b * F + f) * 6;
#pragma unroll
        for (int i = 0; i < 6; ++i) out[i] = g[i];
    }
}

__global__ void __launch_bounds__(128)
sil_vertex_grad_kernel(int V, int F, int H, int W, const float *__restrict__ verts, const int *__restrict__ faces,
                       const int *__restrict__ adj_off, const int *__restrict__ adj_face, const float *__restrict__ cams,
                       const float *__restrict__ fgrad, float *__restrict__ d_verts)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (v >= V) return;
    float gx = 0.f, gy = 0.f;
    for (int k = adj_off[v], prev = -1; k < adj_off[v + 1]; ++k) {
        const int f = adj_face[k];
        if (f == prev) continue;             // a face listed twice at v has two equal corners: zero area, zero gradient
        prev = f;
        const int i = faces[3 * (size_t)f] == v ? 0 : faces[3 * (size_t)f + 1] == v ? 1 : 2;
        const float *gf = fgrad + ((size_t)b * F + f) * 6;
        gx += gf[2 * i];
        gy += gf[2 * i + 1];
    }
    float *out = d_verts + ((size_t)b * V + v) * 3;
    if (gx == 0.f && gy == 0.f) { out[0] = out[1] = out[2] = 0.f; return; }
    // pix_x = ((hx / (hw + 1e-7) + 1) W - 1) / 2, pix_y likewise with hy and H; coordinate k enters row r through proj[4 k + r]
    const float *X = verts + ((size_t)b * V + v) * 3, *proj = cams + (size_t)b * kCamStride + 16;
    const float hx = mesh::xf_row(proj, 0, X[0], X[1], X[2]), hy = mesh::xf_row(proj, 1, X[0], X[1], X[2]);
    const float p_w = 1.f / (mesh::xf_row(proj, 3, X[0], X[1], X[2]) + 0.0000001f);
    const float sx = gx * 0.5f * (float)W * p_w, sy = gy * 0.5f * (float)H * p_w;
#pragma unroll
    for (int k = 0; k < 3; ++k)
        out[k] = sx * (proj[4 * k] - hx * p_w * proj[4 * k + 3]) + sy * (proj[4 * k + 1] - hy * p_w * proj[4 * k + 3]);
}

struct SilWs {
    int4 *boxes;
    FaceXY *xy;
    float *pix, *partial, *fgrad;
    size_t total;
};

SilWs carve(void *p, int B, int F, int H, int W)
{
    Carver c(p);
    SilWs w;
    w.boxes = c.take<int4>((size_t)B * F);
    w.xy = c.take<FaceXY>((size_t)B * F);
    w.pix = c.take<float>((size_t)B * H * W);
    w.partial = c.take<float>((size_t)B * cdiv(H, kTile) * cdiv(W, kTile));
    w.fgrad = c.take<float>((size_t)B * F * 6);
    w.total = c.used();
    return w;
}

int check_args(const char *who, int B, int V, int F, int H, int W, float sigma)
{
    GA_REQUIRE(B >= 1 && B <= kMaxB, "%s: batch %d outside [1, %d]", who, B, kMaxB);
    GA_REQUIRE(V > 0 && V <= (1 << 24) && F >= 0 && F <= (1 << 24), "%s: bad vertex / face count %d / %d", who, V, F);
    GA_REQUIRE(H >= 1 && H <= kMaxSide && W >= 1 && W <= kMaxSide, "%s: frame %d x %d outside [1, %d]^2", who, H, W, kMaxSide);
    GA_REQUIRE(sigma > 0.f && isfinite(sigma), "%s: sigma %g is not a positive number", who, (double)sigma);
    return GA_OK;
}

int launch_setup_and_tiles(int B, int V, int F, int H, int W, float sigma, const float *verts, const int *faces, const float *cams,
                           const unsigned char *mask, const float *w, const SilWs &ws, float *sil, float *partial, float *grad_pix,
                           cudaStream_t stream)
{
    const float trunc_d2 = sigma * kLnInvEps, inv_sigma = 1.f / sigma;
    if (F > 0) {
        { ProfScope _ps("sil_setup_kernel", stream);
          sil_setup_kernel<<<dim3(cdiv(F, 128), B), 128, 0, stream>>>(F, V, H, W, trunc_d2, verts, faces, cams, ws.boxes, ws.xy); }
        GA_CHECK_LAUNCH("sil_setup_kernel");
    }
    { ProfScope _ps("sil_tile_kernel", stream);
      sil_tile_kernel<<<dim3(cdiv(W, kTile) * cdiv(H, kTile), B), kThreads, 0, stream>>>(F, H, W, inv_sigma, trunc_d2, ws.boxes, ws.xy, mask,
                                                                                          w, sil, partial, grad_pix); }
    GA_CHECK_LAUNCH("sil_tile_kernel");
    return GA_OK;
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" size_t ga_silhouette_workspace_bytes(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W)
{
    if (B < 0 || V < 0 || F < 0 || H < 0 || W < 0) return 0;
    return carve(nullptr, B, F, H, W).total;
}

extern "C" int ga_silhouette_forward(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, float sigma, const float *verts,
                                     const int32_t *faces, const float *cams, const uint8_t *mask_u8, void *workspace, float *sil, float *loss,
                                     void *stream_)
{
    if (int rc = check_args("ga_silhouette_forward", B, V, F, H, W, sigma)) return rc;
    GA_REQUIRE(verts && cams && workspace && sil && (F == 0 || faces) && (!mask_u8 || loss), "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const SilWs ws = carve(workspace, B, F, H, W);
    if (int rc = launch_setup_and_tiles(B, V, F, H, W, sigma, verts, faces, cams, mask_u8, nullptr, ws, sil, mask_u8 ? ws.partial : nullptr,
                                        nullptr, stream))
        return rc;
    if (mask_u8) {
        { ProfScope _ps("sil_loss_kernel", stream);
          sil_loss_kernel<<<B, kThreads, 0, stream>>>(cdiv(H, kTile) * cdiv(W, kTile), H, W, ws.partial, loss); }
        GA_CHECK_LAUNCH("sil_loss_kernel");
    }
    return GA_OK;
}

extern "C" int ga_silhouette_backward(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, float sigma, const float *verts,
                                      const int32_t *faces, const int32_t *adj_offsets, const int32_t *adj_faces, const float *cams,
                                      const uint8_t *mask_u8, const float *w, void *workspace, float *d_verts, void *stream_)
{
    if (int rc = check_args("ga_silhouette_backward", B, V, F, H, W, sigma)) return rc;
    GA_REQUIRE(verts && cams && mask_u8 && w && workspace && d_verts && adj_offsets && (F == 0 || (faces && adj_faces)),
               "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const SilWs ws = carve(workspace, B, F, H, W);
    if (int rc = launch_setup_and_tiles(B, V, F, H, W, sigma, verts, faces, cams, mask_u8, w, ws, nullptr, nullptr, ws.pix, stream)) return rc;
    if (F > 0) {
        { ProfScope _ps("sil_face_grad_kernel", stream);
          sil_face_grad_kernel<<<dim3(cdiv(F, 8), B), 256, 0, stream>>>(F, H, W, 1.f / sigma, sigma * kLnInvEps, ws.boxes, ws.xy, ws.pix,
                                                                         ws.fgrad); }
        GA_CHECK_LAUNCH("sil_face_grad_kernel");
    }
    { ProfScope _ps("sil_vertex_grad_kernel", stream);
      sil_vertex_grad_kernel<<<dim3(cdiv(V, 128), B), 128, 0, stream>>>(V, F, H, W, verts, faces, adj_offsets, adj_faces, cams, ws.fgrad,
                                                                         d_verts); }
    GA_CHECK_LAUNCH("sil_vertex_grad_kernel");
    return GA_OK;
}
