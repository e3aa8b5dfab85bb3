// Stage-2 input position maps on the device: posed SMPL / SMPL-X mesh vertices and their backward, the UV-space coverage layout, and
// the per-frame fill and its backward.
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
#include "fixed_raster.cuh"
#include "smpl_math.cuh"

namespace ga {
namespace {

constexpr int kMaxB = 8;
constexpr int kVertsPerCta = 32;
constexpr int kCols = 3 * kVertsPerCta;          // posedirs columns per CTA
constexpr int kRowGroups = 4;                    // posedirs rows split over this many thread groups
constexpr int kVertThreads = kCols * kRowGroups;
constexpr int kNoFace = 0x7f7f7f7f;                // face_id before the raster pass: every byte 0x7f (one memset)
constexpr int kMaxS = 512;

// The pose phase of vertex posing, forward and backward alike: the pose features feat[b] (R_j - I of every joint but the root) and
// the rest-relative joint transforms A[b] of B <= 8 frames.  The B x kJ (frame, joint) pairs are spread over the CTA's kThreads
// threads, and each pair forms its own product of ancestors, so a frame's result does not depend on the batch it is in.  L holds
// the local transforms; it is dead on return.
template <int kJ, int kThreads>
__device__ __forceinline__ void pose_phase(int B, const float *__restrict__ pose, const float *__restrict__ rest_pose,
                                           const float *__restrict__ J, float (*L)[kJ][12], float (*A)[kJ][12],
                                           float (*feat)[Body<kJ>::kFeat])
{
    for (int i = threadIdx.x; i < B * kJ; i += kThreads) {
        const int b = i / kJ, j = i % kJ;
        float r[3], R[9], th;
        joint_axis_angle<kJ>(pose, rest_pose, b, j, r);
        rodrigues(r, R, &th);
        local_transform<kJ>(R, J, j, L[b][j]);
        if (j > 0) {
#pragma unroll
            for (int k = 0; k < 9; ++k) feat[b][(j - 1) * 9 + k] = R[k] - ((k % 4 == 0) ? 1.f : 0.f);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < B * kJ; i += kThreads) {
        const int b = i / kJ, j = i % kJ;
        float G[12];
        chain_product<kJ>(L[b], j, G);
        rest_relative(G, J, j, A[b][j]);
    }
    __syncthreads();
}

// T_v = sum_j w_vj A_j: the blended transform of a vertex with skinning weights w [kJ], from one frame's A
template <int kJ>
__device__ __forceinline__ void blend_transform(const float *__restrict__ w, const float (*A)[12], float T[12])
{
#pragma unroll
    for (int q = 0; q < 12; ++q) T[q] = 0.f;
    for (int j = 0; j < kJ; ++j) {
        const float wj = w[j];
#pragma unroll
        for (int q = 0; q < 12; ++q) T[q] = fmaf(wj, A[j][q], T[q]);
    }
}

// 28.1 KB for SMPL, 56.4 KB for SMPL-X (above the 48 KB of static shared memory: dynamic, with the opt-in).  The local transforms
// are dead once A is formed, so the row-group partial sums reuse their space.
template <int kJ> struct VertSmem {
    float A[kMaxB][kJ][12];
    float feat[kMaxB][Body<kJ>::kFeat];
    union {
        float L[kMaxB][kJ][12];
        float part[kRowGroups][kMaxB][kCols];
    } u;
};

// Posed vertices of B <= 8 frames.  Every CTA forms the B frames' pose features and joint transforms A (pose_phase), then streams its
// 96 columns of posedirs [kFeat, 3V] ONCE for all B frames (four row groups, reduced in shared memory), then skins its 32 vertices.
template <int kJ>
__global__ void __launch_bounds__(kVertThreads)
vertices_kernel(int B, int V, const float *__restrict__ pose /*[B,3 kTrained]*/, const float *__restrict__ rest_pose /*[B,3 (kJ-kTrained)]*/,
                const float *__restrict__ transl /*[B,3]*/, const float *__restrict__ J /*[kJ,3]*/,
                const float *__restrict__ v_shaped /*[V,3]*/, const float *__restrict__ posedirs /*[kFeat,3V]*/,
                const float *__restrict__ weights /*[V,kJ]*/, float *__restrict__ verts /*[B,V,3]*/)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    VertSmem<kJ> &sm = *reinterpret_cast<VertSmem<kJ> *>(smem_raw);
    const int tid = threadIdx.x;
    pose_phase<kJ, kVertThreads>(B, pose, rest_pose, J, sm.u.L, sm.A, sm.feat);     // L is dead from here on: part may overwrite it

    // pose blend shapes: column k of posedirs, rows rg, rg + 4, ...; one accumulator per frame
    const int col = tid % kCols, rg = tid / kCols;
    const long long ncol = 3LL * V;
    const long long k = (long long)blockIdx.x * kCols + col;
    float acc[kMaxB];
#pragma unroll
    for (int b = 0; b < kMaxB; ++b) acc[b] = 0.f;
    if (k < ncol) {
#pragma unroll 4
        for (int r = rg; r < Body<kJ>::kFeat; r += kRowGroups) {
            const float pd = __ldg(posedirs + (long long)r * ncol + k);
#pragma unroll
            for (int b = 0; b < kMaxB; ++b)
                if (b < B) acc[b] = fmaf(sm.feat[b][r], pd, acc[b]);
        }
    }
#pragma unroll
    for (int b = 0; b < kMaxB; ++b)
        if (b < B) sm.u.part[rg][b][col] = acc[b];
    __syncthreads();

    // skinning: x = T_v [v_posed; 1] + transl
    for (int i = tid; i < kVertsPerCta * B; i += kVertThreads) {
        const int vl = i % kVertsPerCta, b = i / kVertsPerCta;
        const int v = blockIdx.x * kVertsPerCta + vl;
        if (v >= V) continue;
        float x[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float off = 0.f;
#pragma unroll
            for (int g = 0; g < kRowGroups; ++g) off += sm.u.part[g][b][vl * 3 + c];
            x[c] = v_shaped[(size_t)v * 3 + c] + off;
        }
        float T[12];
        blend_transform<kJ>(weights + (size_t)v * kJ, sm.A[b], T);
        float *o = verts + ((size_t)b * V + v) * 3;
#pragma unroll
        for (int r = 0; r < 3; ++r)
            o[r] = T[r * 4 + 0] * x[0] + T[r * 4 + 1] * x[1] + T[r * 4 + 2] * x[2] + T[r * 4 + 3] + transl[b * 3 + r];
    }
}

// out[t, j] = sum_i bary[t, i] W[faces[face_id[t], i], j] (fp32, i in order), 0 where face_id is -1: the texel skinning weights of
// the reference's gen_lbs_weight_from_ori (utils/general_utils.py:245-259).  One thread per output element, so the stores coalesce.
__global__ void __launch_bounds__(256)
posmap_weights_kernel(int n, int J, const float *__restrict__ W, const int *__restrict__ faces, const int *__restrict__ face_id,
                      const float *__restrict__ bary, float *__restrict__ out)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int t = e / J, j = e - t * J;
    const int f = face_id[t];
    float o = 0.f;
    if (f >= 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) o = fmaf(bary[(size_t)t * 3 + i], W[(size_t)faces[(size_t)f * 3 + i] * J + j], o);
    }
    out[e] = o;
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
        s.x[i] = s.ok ? snap_fixed((double)u * scale) : 0;
        s.y[i] = s.ok ? snap_fixed((double)v * scale) : 0;
    }
    return s;
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

// ---- backward of vertex posing (ga_smpl_vertices_backward / ga_smplx_vertices_backward)
//
// With g_v = d_verts[b,v], x_v = v_shaped_v + posedirs^T feat (the blend-shaped vertex) and T_v = sum_j w_vj A_j:
//   d_transl = sum_v g_v,   d_A_j = sum_v w_vj g_v [x_v; 1]^T,   d_feat[r] = sum_{v,c} posedirs[r, 3v+c] (T_v[:, :3]^T g_v)_c.
// Pass 1 (one CTA per 32 vertices, as the forward) streams posedirs once for all B frames: it needs T_v^T g_v (from A) before the
// stream and x_v (from the stream) after it.  Each CTA writes its per-frame sums [d_A | d_feat | d_transl] to its own workspace slot.
// Pass 2 (one CTA per frame) adds the slots in CTA order, then runs the joint chain and the Rodrigues map backwards.  No atomics:
// the results are bit-reproducible, and a frame's sums never mix with another frame's, so they do not depend on the batch.
constexpr int kBwdThreads = 256;
constexpr int kBwdWarps = kBwdThreads / 32;

// per-frame sums of one CTA: d_A [J,12], d_feat [kFeat], d_transl [3]
template <int kJ> constexpr int bwd_sums() { return kJ * 12 + Body<kJ>::kFeat + 3; }

template <int kJ> struct VertBwdSmem {
    float A[kMaxB][kJ][12];
    float feat[kMaxB][Body<kJ>::kFeat];
    float g[kMaxB][kCols];           // d_verts of the CTA's 32 vertices
    float dx[kMaxB][kCols];          // T_v[:, :3]^T g_v
    float x[kMaxB][kCols];           // blend-shaped vertices
    union {
        float L[kMaxB][kJ][12];
        float part[kBwdWarps][kMaxB][kCols];
        float gx[kMaxB][kVertsPerCta][12];     // g_v [x_v; 1]^T
    } u;
};

template <int kJ> struct VertFinishSmem {
    float sums[bwd_sums<kJ>()];
    float L[kJ][12], G[kJ][12], dG[kJ][12], dR[kJ][9];
};

template <int kJ>
__global__ void __launch_bounds__(kBwdThreads, 1)
vertices_bwd_kernel(int B, int V, const float *__restrict__ pose, const float *__restrict__ rest_pose, const float *__restrict__ J,
                    const float *__restrict__ v_shaped, const float *__restrict__ posedirs, const float *__restrict__ weights,
                    const float *__restrict__ d_verts, float *__restrict__ sums /*[ctas][B][bwd_sums]*/)
{
    constexpr int kF = Body<kJ>::kFeat, kN = bwd_sums<kJ>();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    VertBwdSmem<kJ> &sm = *reinterpret_cast<VertBwdSmem<kJ> *>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long ncol = 3LL * V, k0 = (long long)blockIdx.x * kCols;
    float *out = sums + (size_t)blockIdx.x * B * kN;

    for (int i = tid; i < B * kCols; i += kBwdThreads) {
        const int b = i / kCols, col = i % kCols;
        sm.g[b][col] = (k0 + col < ncol) ? d_verts[(size_t)b * ncol + k0 + col] : 0.f;
    }
    pose_phase<kJ, kBwdThreads>(B, pose, rest_pose, J, sm.u.L, sm.A, sm.feat);     // L is dead from here on

    // dx_v = T_v[:, :3]^T g_v
    for (int i = tid; i < B * kVertsPerCta; i += kBwdThreads) {
        const int b = i / kVertsPerCta, vl = i % kVertsPerCta;
        const int v = blockIdx.x * kVertsPerCta + vl;
        float d[3] = {0.f, 0.f, 0.f};
        if (v < V) {
            float T[12];
            blend_transform<kJ>(weights + (size_t)v * kJ, sm.A[b], T);
            const float *g = sm.g[b] + vl * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) d[c] = T[c] * g[0] + T[4 + c] * g[1] + T[8 + c] * g[2];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) sm.dx[b][vl * 3 + c] = d[c];
    }
    __syncthreads();

    // posedirs, once for all frames: warp w takes rows w, w + 8, ...; lane takes columns lane, lane + 32, lane + 64.  Per row, the
    // warp sums pd dx over its 96 columns (d_feat) and every lane accumulates feat pd into its columns (the forward's offsets).
    float dxr[kMaxB][3], off[kMaxB][3];
#pragma unroll
    for (int b = 0; b < kMaxB; ++b)
#pragma unroll
        for (int m = 0; m < 3; ++m) { dxr[b][m] = (b < B) ? sm.dx[b][lane + 32 * m] : 0.f; off[b][m] = 0.f; }
    for (int r = warp; r < kF; r += kBwdWarps) {
        float pd[3];
#pragma unroll
        for (int m = 0; m < 3; ++m) {
            const long long k = k0 + lane + 32 * m;
            pd[m] = (k < ncol) ? __ldg(posedirs + (long long)r * ncol + k) : 0.f;
        }
#pragma unroll
        for (int b = 0; b < kMaxB; ++b) {
            if (b < B) {
                const float f = sm.feat[b][r];
                float s = pd[0] * dxr[b][0] + pd[1] * dxr[b][1] + pd[2] * dxr[b][2];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                if (lane == b) out[(size_t)b * kN + kJ * 12 + r] = s;
#pragma unroll
                for (int m = 0; m < 3; ++m) off[b][m] = fmaf(f, pd[m], off[b][m]);
            }
        }
    }
#pragma unroll
    for (int b = 0; b < kMaxB; ++b)
        if (b < B)
#pragma unroll
            for (int m = 0; m < 3; ++m) sm.u.part[warp][b][lane + 32 * m] = off[b][m];
    __syncthreads();
    for (int i = tid; i < B * kCols; i += kBwdThreads) {
        const int b = i / kCols, col = i % kCols;
        float o = 0.f;
#pragma unroll
        for (int w = 0; w < kBwdWarps; ++w) o += sm.u.part[w][b][col];
        sm.x[b][col] = (k0 + col < ncol) ? v_shaped[k0 + col] + o : 0.f;
    }
    __syncthreads();        // part is dead from here on
    for (int i = tid; i < B * kVertsPerCta; i += kBwdThreads) {
        const int b = i / kVertsPerCta, vl = i % kVertsPerCta;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float g = sm.g[b][vl * 3 + r];
            sm.u.gx[b][vl][r * 4 + 0] = g * sm.x[b][vl * 3 + 0];
            sm.u.gx[b][vl][r * 4 + 1] = g * sm.x[b][vl * 3 + 1];
            sm.u.gx[b][vl][r * 4 + 2] = g * sm.x[b][vl * 3 + 2];
            sm.u.gx[b][vl][r * 4 + 3] = g;
        }
    }
    __syncthreads();
    const int vbase = blockIdx.x * kVertsPerCta, nv = min(kVertsPerCta, V - vbase);
    for (int i = tid; i < B * kJ * 12; i += kBwdThreads) {
        const int b = i / (kJ * 12), jq = i % (kJ * 12), j = jq / 12, q = jq % 12;
        float s = 0.f;
        for (int vl = 0; vl < nv; ++vl) s = fmaf(weights[(size_t)(vbase + vl) * kJ + j], sm.u.gx[b][vl][q], s);
        out[(size_t)b * kN + jq] = s;
    }
    for (int i = tid; i < B * 3; i += kBwdThreads) {
        const int b = i / 3, c = i % 3;
        float s = 0.f;
        for (int vl = 0; vl < nv; ++vl) s += sm.g[b][vl * 3 + c];
        out[(size_t)b * kN + kJ * 12 + kF + c] = s;
    }
}

// One CTA per frame: add the CTAs' sums in order, then d_A -> d_G -> (joint chain, leaves first) d_L -> d_R (+ d_feat) -> d_pose.
template <int kJ>
__global__ void __launch_bounds__(kBwdThreads)
vertices_bwd_finish_kernel(int B, int ctas, const float *__restrict__ pose, const float *__restrict__ rest_pose,
                           const float *__restrict__ J, const float *__restrict__ sums, float *__restrict__ d_pose, float *__restrict__ d_transl)
{
    constexpr int kF = Body<kJ>::kFeat, kN = bwd_sums<kJ>(), kT = Body<kJ>::kTrained;
    __shared__ VertFinishSmem<kJ> sm;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    for (int e = tid; e < kN; e += kBwdThreads) {
        float s = 0.f;
        for (int c = 0; c < ctas; ++c) s += sums[((size_t)c * B + b) * kN + e];
        sm.sums[e] = s;
    }
    for (int j = tid; j < kJ; j += kBwdThreads) {
        float r[3], R[9], th;
        joint_axis_angle<kJ>(pose, rest_pose, b, j, r);
        rodrigues(r, R, &th);
        local_transform<kJ>(R, J, j, sm.L[j]);
    }
    __syncthreads();
    for (int i = tid; i < kJ * 12; i += kBwdThreads) {
        const int j = i / 12, q = i % 12, rr = q / 4, c = q % 4;
        if (q == 0) chain_product<kJ>(sm.L, j, sm.G[j]);
        // A[:, 3] = G[:, 3] - G[:, :3] J_j
        const float *dA = sm.sums + j * 12;
        sm.dG[j][q] = (c == 3) ? dA[rr * 4 + 3] : dA[rr * 4 + c] - dA[rr * 4 + 3] * J[j * 3 + c];
    }
    __syncthreads();
    if (tid < 32) {
        // G_j = G_p L_j, leaves first (every parent index is below its child's); lane q owns element q of d_G_p, lane < 9 of d_L_j
        for (int j = kJ - 1; j >= 0; --j) {
            const int p = Body<kJ>::parent(j);
            const float *dG = sm.dG[j];
            if (lane < 9) {
                const int rr = lane / 3, k = lane % 3;
                sm.dR[j][lane] = (p < 0) ? dG[rr * 4 + k]
                                         : sm.G[p][rr] * dG[k] + sm.G[p][4 + rr] * dG[4 + k] + sm.G[p][8 + rr] * dG[8 + k];
            }
            if (p >= 0 && lane < 12) {
                const int rr = lane / 4, c = lane % 4;
                const float *L = sm.L[j];
                const float u = (c == 3) ? dG[rr * 4 + 3]
                                         : dG[rr * 4] * L[c * 4] + dG[rr * 4 + 1] * L[c * 4 + 1] + dG[rr * 4 + 2] * L[c * 4 + 2] +
                                               dG[rr * 4 + 3] * L[c * 4 + 3];
                sm.dG[p][lane] += u;
            }
            __syncwarp();
        }
    }
    __syncthreads();
    for (int j = tid; j < kT; j += kBwdThreads) {
        float r[3], gR[9], gr[3];
        joint_axis_angle<kJ>(pose, rest_pose, b, j, r);
#pragma unroll
        for (int k = 0; k < 9; ++k) gR[k] = sm.dR[j][k] + ((j > 0) ? sm.sums[kJ * 12 + (j - 1) * 9 + k] : 0.f);
        rodrigues_bwd(r, gR, gr);
#pragma unroll
        for (int k = 0; k < 3; ++k) d_pose[(size_t)b * 3 * kT + j * 3 + k] = gr[k];
    }
    if (tid < 3) d_transl[b * 3 + tid] = sm.sums[kJ * 12 + kF + tid];
}

// ---- backward of the fill through a vertex -> (texel, corner) CSR
//
// entries hold 3 t + i for texel t whose covering face has the vertex as corner i, in ascending order per vertex.  Built once per
// layout: count (integer atomics), inclusive scan, scatter (a cursor that counts down from each vertex's end to its start), then a
// per-vertex sort, so the order does not depend on the scatter's.
__global__ void __launch_bounds__(256)
posmap_csr_count_kernel(int n, const int *__restrict__ faces, const int *__restrict__ face_id, int *__restrict__ offsets)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int f = face_id[t];
    if (f < 0) return;
#pragma unroll
    for (int i = 0; i < 3; ++i) atomicAdd(offsets + faces[(size_t)f * 3 + i], 1);
}

// one CTA: offsets[v] = count[0] + ... + count[v] (inclusive), offsets[V] = the total
__global__ void __launch_bounds__(1024)
posmap_csr_scan_kernel(int V, int *__restrict__ offsets)
{
    __shared__ int warp_sums[32];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < V; base += 1024) {
        const int i = base + tid;
        int x = (i < V) ? offsets[i] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int w = warp_sums[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            warp_sums[lane] = w;
        }
        __syncthreads();
        const int c = carry;
        x += c + (warp > 0 ? warp_sums[warp - 1] : 0);
        if (i < V) offsets[i] = x;
        __syncthreads();
        if (tid == 1023) carry = x;
        __syncthreads();
    }
    if (tid == 0) offsets[V] = carry;
}

__global__ void __launch_bounds__(256)
posmap_csr_scatter_kernel(int n, const int *__restrict__ faces, const int *__restrict__ face_id, int *__restrict__ offsets,
                          int *__restrict__ entries)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int f = face_id[t];
    if (f < 0) return;
#pragma unroll
    for (int i = 0; i < 3; ++i) entries[atomicSub(offsets + faces[(size_t)f * 3 + i], 1) - 1] = 3 * t + i;
}

// one thread per vertex: heapsort of its entries (any length, no extra memory)
__global__ void __launch_bounds__(256)
posmap_csr_sort_kernel(int V, const int *__restrict__ offsets, int *__restrict__ entries)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    int *a = entries + offsets[v];
    const int n = offsets[v + 1] - offsets[v];
    auto sift = [a](int root, int end) {
        while (2 * root + 1 < end) {
            int c = 2 * root + 1;
            if (c + 1 < end && a[c + 1] > a[c]) ++c;
            if (a[root] >= a[c]) return;
            const int t = a[root]; a[root] = a[c]; a[c] = t;
            root = c;
        }
    };
    for (int i = n / 2 - 1; i >= 0; --i) sift(i, n);
    for (int end = n - 1; end > 0; --end) {
        const int t = a[0]; a[0] = a[end]; a[end] = t;
        sift(0, end);
    }
}

// d_verts[b, v, :] = sum over v's entries (t, i) of bary[t, i] d_out[b, :, t].  One warp per (vertex, frame): lanes stride over the
// entries, then a fixed butterfly; every element of d_verts is written (0 for a vertex no texel uses).
constexpr int kFillBwdWarps = 8;

__global__ void __launch_bounds__(kFillBwdWarps * 32)
posmap_fill_bwd_kernel(int S, int V, const int *__restrict__ offsets, const int *__restrict__ entries, const float *__restrict__ bary,
                       const float *__restrict__ d_out, float *__restrict__ d_verts)
{
    const int v = blockIdx.x * kFillBwdWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31, b = blockIdx.y;
    if (v >= V) return;
    const int n = S * S;
    const float *g = d_out + (size_t)b * 3 * n;
    float a[3] = {0.f, 0.f, 0.f};
    for (int e = offsets[v] + lane; e < offsets[v + 1]; e += 32) {
        const int ti = entries[e], t = ti / 3;
        const float w = bary[ti];
        a[0] = fmaf(w, g[t], a[0]); a[1] = fmaf(w, g[n + t], a[1]); a[2] = fmaf(w, g[2 * n + t], a[2]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int c = 0; c < 3; ++c) a[c] += __shfl_xor_sync(0xffffffffu, a[c], o);
    }
    if (lane < 3) d_verts[((size_t)b * V + v) * 3 + lane] = a[lane];
}

template <int kJ>
int vertices_forward(const char *name, int B, int V, const float *pose, const float *rest_pose, const float *transl, const float *rest_joints,
                     const float *v_shaped, const float *posedirs, const float *weights, float *verts, cudaStream_t stream)
{
    GA_REQUIRE(B >= 0 && B <= kMaxB, "%s: batch %d outside [0, %d]", name, B, kMaxB);
    GA_REQUIRE(V > 0 && V <= (1 << 24), "%s: bad vertex count %d", name, V);
    if (B == 0) return GA_OK;
    GA_REQUIRE(pose && (kJ == kSmplJoints || rest_pose) && transl && rest_joints && v_shaped && posedirs && weights && verts,
               "NULL pointer argument");
    static PerDeviceOnce attr_set;
    if (attr_set.first())
        GA_CHECK_CUDA(cudaFuncSetAttribute(vertices_kernel<kJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VertSmem<kJ>)));
    const char *kernel = kJ == kSmplJoints ? "smpl_vertices_kernel" : "smplx_vertices_kernel";
    { ProfScope _ps(kernel, stream);
      vertices_kernel<kJ><<<cdiv(V, kVertsPerCta), kVertThreads, sizeof(VertSmem<kJ>), stream>>>(B, V, pose, rest_pose, transl, rest_joints,
                                                                                               v_shaped, posedirs, weights, verts); }
    GA_CHECK_LAUNCH(kernel);
    return GA_OK;
}

template <int kJ> size_t vertices_bwd_workspace(int B, int V)
{
    if (B < 1 || B > kMaxB || V < 1 || V > (1 << 24)) return 0;
    return (size_t)cdiv(V, kVertsPerCta) * B * bwd_sums<kJ>() * sizeof(float);
}

template <int kJ>
int vertices_backward(const char *name, int B, int V, const float *pose, const float *rest_pose, const float *rest_joints, const float *v_shaped,
                      const float *posedirs, const float *weights, const float *d_verts, void *workspace, size_t workspace_bytes,
                      float *d_pose, float *d_transl, cudaStream_t stream)
{
    GA_REQUIRE(B >= 1 && B <= kMaxB, "%s: batch %d outside [1, %d]", name, B, kMaxB);
    GA_REQUIRE(V > 0 && V <= (1 << 24), "%s: bad vertex count %d", name, V);
    GA_REQUIRE(pose && (kJ == kSmplJoints || rest_pose) && rest_joints && v_shaped && posedirs && weights && d_verts && workspace && d_pose && d_transl,
               "%s: NULL pointer argument", name);
    const size_t need = vertices_bwd_workspace<kJ>(B, V);
    GA_REQUIRE(workspace_bytes >= need, "%s: workspace of %zu bytes, %zu needed", name, workspace_bytes, need);
    GA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 3) == 0, "%s: workspace must be 4-byte aligned", name);
    static PerDeviceOnce attr_set;
    if (attr_set.first())
        GA_CHECK_CUDA(cudaFuncSetAttribute(vertices_bwd_kernel<kJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VertBwdSmem<kJ>)));
    const int ctas = cdiv(V, kVertsPerCta);
    float *sums = static_cast<float *>(workspace);
    { ProfScope _ps(kJ == kSmplJoints ? "smpl_vertices_bwd_kernel" : "smplx_vertices_bwd_kernel", stream);
      vertices_bwd_kernel<kJ><<<ctas, kBwdThreads, sizeof(VertBwdSmem<kJ>), stream>>>(B, V, pose, rest_pose, rest_joints, v_shaped,
                                                                                      posedirs, weights, d_verts, sums); }
    GA_CHECK_LAUNCH("vertices_bwd_kernel");
    { ProfScope _ps(kJ == kSmplJoints ? "smpl_vertices_bwd_finish_kernel" : "smplx_vertices_bwd_finish_kernel", stream);
      vertices_bwd_finish_kernel<kJ><<<B, kBwdThreads, 0, stream>>>(B, ctas, pose, rest_pose, rest_joints, sums, d_pose, d_transl); }
    GA_CHECK_LAUNCH("vertices_bwd_finish_kernel");
    return GA_OK;
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_smpl_vertices(int32_t B, int32_t V, const float *pose, const float *transl, const float *rest_joints,
                                const float *v_shaped, const float *posedirs, const float *weights, float *verts, void *stream_)
{
    return vertices_forward<kSmplJoints>("ga_smpl_vertices", B, V, pose, nullptr, transl, rest_joints, v_shaped, posedirs, weights, verts,
                                         static_cast<cudaStream_t>(stream_));
}

extern "C" int ga_smplx_vertices(int32_t B, int32_t V, const float *pose, const float *rest_pose, const float *transl, const float *rest_joints,
                                 const float *v_shaped, const float *posedirs, const float *weights, float *verts, void *stream_)
{
    return vertices_forward<kSmplxJoints>("ga_smplx_vertices", B, V, pose, rest_pose, transl, rest_joints, v_shaped, posedirs, weights, verts,
                                          static_cast<cudaStream_t>(stream_));
}

extern "C" int ga_posmap_weights(int32_t S, int32_t J, const float *weights, const int32_t *faces, const int32_t *face_id, const float *bary,
                                 float *out, void *stream_)
{
    GA_REQUIRE(S >= 1 && S <= kMaxS, "ga_posmap_weights: map size %d outside [1, %d]", S, kMaxS);
    GA_REQUIRE(J == kSmplJoints || J == kSmplxJoints, "ga_posmap_weights: joint count %d is neither %d (SMPL) nor %d (SMPL-X)", J, kSmplJoints, kSmplxJoints);
    GA_REQUIRE(weights && faces && face_id && bary && out, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int n = S * S * J;
    { ProfScope _ps("posmap_weights_kernel", stream);
      posmap_weights_kernel<<<cdiv(n, 256), 256, 0, stream>>>(n, J, weights, faces, face_id, bary, out); }
    GA_CHECK_LAUNCH("posmap_weights_kernel");
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

extern "C" size_t ga_smpl_vertices_backward_workspace_bytes(int32_t B, int32_t V) { return vertices_bwd_workspace<kSmplJoints>(B, V); }
extern "C" size_t ga_smplx_vertices_backward_workspace_bytes(int32_t B, int32_t V) { return vertices_bwd_workspace<kSmplxJoints>(B, V); }

extern "C" int ga_smpl_vertices_backward(int32_t B, int32_t V, const float *pose, const float *rest_joints, const float *v_shaped,
                                         const float *posedirs, const float *weights, const float *d_verts, void *workspace,
                                         size_t workspace_bytes, float *d_pose, float *d_transl, void *stream_)
{
    return vertices_backward<kSmplJoints>("ga_smpl_vertices_backward", B, V, pose, nullptr, rest_joints, v_shaped, posedirs, weights, d_verts,
                                      workspace, workspace_bytes, d_pose, d_transl, static_cast<cudaStream_t>(stream_));
}

extern "C" int ga_smplx_vertices_backward(int32_t B, int32_t V, const float *pose, const float *rest_pose, const float *rest_joints,
                                          const float *v_shaped, const float *posedirs, const float *weights, const float *d_verts,
                                          void *workspace, size_t workspace_bytes, float *d_pose, float *d_transl, void *stream_)
{
    return vertices_backward<kSmplxJoints>("ga_smplx_vertices_backward", B, V, pose, rest_pose, rest_joints, v_shaped, posedirs, weights,
                                       d_verts, workspace, workspace_bytes, d_pose, d_transl, static_cast<cudaStream_t>(stream_));
}

extern "C" int ga_posmap_vertex_csr(int32_t S, int32_t V, const int32_t *faces, const int32_t *face_id, int32_t *offsets, int32_t *entries,
                                    void *stream_)
{
    GA_REQUIRE(S >= 1 && S <= kMaxS, "ga_posmap_vertex_csr: map size %d outside [1, %d]", S, kMaxS);
    GA_REQUIRE(V > 0 && V <= (1 << 24), "ga_posmap_vertex_csr: bad vertex count %d", V);
    GA_REQUIRE(faces && face_id && offsets && entries, "ga_posmap_vertex_csr: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int n = S * S;
    GA_CHECK_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int32_t) * ((size_t)V + 1), stream));
    { ProfScope _ps("posmap_csr_count_kernel", stream);
      posmap_csr_count_kernel<<<cdiv(n, 256), 256, 0, stream>>>(n, faces, face_id, offsets); }
    GA_CHECK_LAUNCH("posmap_csr_count_kernel");
    { ProfScope _ps("posmap_csr_scan_kernel", stream); posmap_csr_scan_kernel<<<1, 1024, 0, stream>>>(V, offsets); }
    GA_CHECK_LAUNCH("posmap_csr_scan_kernel");
    { ProfScope _ps("posmap_csr_scatter_kernel", stream);
      posmap_csr_scatter_kernel<<<cdiv(n, 256), 256, 0, stream>>>(n, faces, face_id, offsets, entries); }
    GA_CHECK_LAUNCH("posmap_csr_scatter_kernel");
    { ProfScope _ps("posmap_csr_sort_kernel", stream); posmap_csr_sort_kernel<<<cdiv(V, 256), 256, 0, stream>>>(V, offsets, entries); }
    GA_CHECK_LAUNCH("posmap_csr_sort_kernel");
    return GA_OK;
}

extern "C" int ga_posmap_fill_backward(int32_t B, int32_t S, int32_t V, const int32_t *csr_offsets, const int32_t *csr_entries,
                                       const float *bary, const float *d_out, float *d_verts, void *stream_)
{
    GA_REQUIRE(B >= 1 && B <= kMaxB, "ga_posmap_fill_backward: batch %d outside [1, %d]", B, kMaxB);
    GA_REQUIRE(S >= 1 && S <= kMaxS, "ga_posmap_fill_backward: map size %d outside [1, %d]", S, kMaxS);
    GA_REQUIRE(V > 0 && V <= (1 << 24), "ga_posmap_fill_backward: bad vertex count %d", V);
    GA_REQUIRE(csr_offsets && csr_entries && bary && d_out && d_verts, "ga_posmap_fill_backward: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("posmap_fill_bwd_kernel", stream);
      posmap_fill_bwd_kernel<<<dim3(cdiv(V, kFillBwdWarps), B), kFillBwdWarps * 32, 0, stream>>>(S, V, csr_offsets, csr_entries, bary, d_out,
                                                                                                  d_verts); }
    GA_CHECK_LAUNCH("posmap_fill_bwd_kernel");
    return GA_OK;
}
