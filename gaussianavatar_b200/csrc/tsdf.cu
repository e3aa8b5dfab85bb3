// Mesh extraction from depth passes: truncated signed distance fusion of B <= 8 views per launch into a regular grid, and marching
// tetrahedra on the Kuhn split of every grid cube.  See DESIGN.md §2 (defined here) for the fusion rules and §4 for the layout.
//
//   tsdf_integrate_kernel  per sample (x fastest): projects the sample as the Gaussian preprocess projects a mean (mesh_project.cuh),
//                          takes the nearest pixel and folds the launch's views into the sample's state in view order, so the state
//                          is read and written once per launch and the result does not depend on how the views are split into
//                          launches.  No atomics.
//   tsdf_count_kernel      per grid point p: the crossing edges p owns (p, p + d), d in {x, y, z, xy, xz, yz, xyz}, as a 7-bit mask,
//                          and the triangles of the cube whose lowest corner is p.  Two CUB exclusive scans turn the counts into
//                          output offsets.
//   tsdf_emit_kernel       per grid point p: its vertices (ordered by owner, then slot) and its cube's triangles (ordered by cube,
//                          tetrahedron, triangle); the id of the vertex on edge (q, slot) is voff[q] + the crossing slots of q below
//                          it.  Nothing is written past the capacities given.
//
// The six tetrahedra of a cube, (p, p + e_a, p + e_a + e_b, p + (1,1,1)) for the six orders (a, b, c) of the axes, split every cube
// along its main diagonal in the same way, so two cubes split their shared face along the same diagonal and the surface is a closed
// 2-manifold wherever the outer layer of the grid is outside.  The triangle table is generated below from one rule.
#include <cub/cub.cuh>

#include "common.cuh"
#include "mesh_project.cuh"

namespace ga {
namespace {

constexpr int kMaxViews = 8;
constexpr int kMinSide = 2, kMaxSide = 512;
constexpr int kMaxImageSide = 16384;
constexpr float kZcull = 0.2f;          // the preprocess's near cull (raster.cu)
constexpr int kPlanes = 7;              // sdf, weight, carve, r, g, b sums, colour weight

// ---- the case table, generated from one rule ---------------------------------------------------------------------------------------
// Cube corner c is at p + (c & 1, (c >> 1) & 1, (c >> 2) & 1).  Tetrahedron t visits corners 0, e_a, e_a + e_b, 7 for the axis order
// kPerm[t].  Local edge e joins tetrahedron vertices kEdgeV[e].  For a sign pattern (bit v: vertex v is inside) the crossing edges
// form one triangle (one or three vertices inside) or a quad (two inside, a, b; outside c, d: the cycle ac, ad, bd, bc, split along
// ac-bd).  Each triangle is wound so that its normal, evaluated at the edge midpoints, points from the inside vertices' centroid to
// the outside vertices'.
constexpr int kPerm[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
constexpr int kEdgeV[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
constexpr int kSlotOfMask[8] = {-1, 0, 1, 3, 2, 4, 5, 6};   // d = x, y, z, xy, xz, yz, xyz -> slot 0..6
__host__ __device__ constexpr int mask_of_slot(int s) { return s < 3 ? 1 << s : s == 3 ? 3 : s == 4 ? 5 : s == 5 ? 6 : 7; }

struct TetTable {
    signed char ntri[6][16];
    signed char edge[6][16][6];      // triangles' local edges, three per triangle
    unsigned char corner[6][4];      // cube corner of each tetrahedron vertex
    unsigned char owner[6][6];       // cube corner owning each local edge (its lower end)
    unsigned char slot[6][6];        // the edge's slot at its owner
};

constexpr int tet_corner(int t, int v)
{
    return v == 0 ? 0 : v == 1 ? (1 << kPerm[t][0]) : v == 2 ? ((1 << kPerm[t][0]) | (1 << kPerm[t][1])) : 7;
}

constexpr int local_edge(int i, int j)
{
    const int a = i < j ? i : j, b = i < j ? j : i;
    for (int e = 0; e < 6; ++e)
        if (kEdgeV[e][0] == a && kEdgeV[e][1] == b) return e;
    return -1;
}

constexpr TetTable build_table()
{
    TetTable T{};
    for (int t = 0; t < 6; ++t) {
        int pos[4][3] = {};
        for (int v = 0; v < 4; ++v) {
            const int c = tet_corner(t, v);
            T.corner[t][v] = (unsigned char)c;
            for (int a = 0; a < 3; ++a) pos[v][a] = (c >> a) & 1;
        }
        for (int e = 0; e < 6; ++e) {
            const int lo = tet_corner(t, kEdgeV[e][0]), hi = tet_corner(t, kEdgeV[e][1]);   // lo is below hi on every axis
            T.owner[t][e] = (unsigned char)lo;
            T.slot[t][e] = (unsigned char)kSlotOfMask[hi ^ lo];
        }
        for (int c = 0; c < 16; ++c) {
            int in[4] = {}, out[4] = {}, ni = 0, no = 0;
            for (int v = 0; v < 4; ++v) {
                if ((c >> v) & 1) in[ni++] = v;
                else out[no++] = v;
            }
            int tris[2][3] = {}, nt = 0;
            if (ni == 1 || ni == 3) {
                const int lone = ni == 1 ? in[0] : out[0];
                const int *rest = ni == 1 ? out : in;
                tris[0][0] = local_edge(lone, rest[0]); tris[0][1] = local_edge(lone, rest[1]); tris[0][2] = local_edge(lone, rest[2]);
                nt = 1;
            } else if (ni == 2) {
                const int ac = local_edge(in[0], out[0]), ad = local_edge(in[0], out[1]), bd = local_edge(in[1], out[1]),
                          bc = local_edge(in[1], out[0]);
                tris[0][0] = ac; tris[0][1] = ad; tris[0][2] = bd;
                tris[1][0] = ac; tris[1][1] = bd; tris[1][2] = bc;
                nt = 2;
            }
            for (int k = 0; k < nt; ++k) {
                int P[3][3] = {};                         // twice the edge midpoints
                for (int q = 0; q < 3; ++q)
                    for (int a = 0; a < 3; ++a) P[q][a] = pos[kEdgeV[tris[k][q]][0]][a] + pos[kEdgeV[tris[k][q]][1]][a];
                const int u[3] = {P[1][0] - P[0][0], P[1][1] - P[0][1], P[1][2] - P[0][2]};
                const int w[3] = {P[2][0] - P[0][0], P[2][1] - P[0][1], P[2][2] - P[0][2]};
                const int n[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
                int o[3] = {};                            // ni * no * (centroid(outside) - centroid(inside))
                for (int a = 0; a < 3; ++a) {
                    for (int q = 0; q < no; ++q) o[a] += ni * pos[out[q]][a];
                    for (int q = 0; q < ni; ++q) o[a] -= no * pos[in[q]][a];
                }
                if (n[0] * o[0] + n[1] * o[1] + n[2] * o[2] < 0) {
                    const int s = tris[k][1]; tris[k][1] = tris[k][2]; tris[k][2] = s;
                }
                for (int q = 0; q < 3; ++q) T.edge[t][c][3 * k + q] = (signed char)tris[k][q];
            }
            T.ntri[t][c] = (signed char)nt;
        }
    }
    return T;
}

__constant__ TetTable c_table = build_table();

// ---- state --------------------------------------------------------------------------------------------------------------------
struct Grid {
    int nx, ny, nz;
    long long N;
    float ox, oy, oz, voxel, trunc;
};

struct State {
    float *sdf; int *weight; int *carve; float *r, *g, *b; int *cw;
};

__host__ __device__ inline State state_of(void *base, long long N)
{
    float *f = static_cast<float *>(base);
    int *i = static_cast<int *>(base);
    return State{f, i + N, i + 2 * N, f + 3 * N, f + 4 * N, f + 5 * N, i + 6 * N};
}

__global__ void __launch_bounds__(256)
tsdf_integrate_kernel(Grid G, int B, int H, int W, const float *__restrict__ cams, const float *__restrict__ depth,
                      const float *__restrict__ image, const float *__restrict__ final_T, State S)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= G.N) return;
    const int i = (int)(idx % G.nx), j = (int)((idx / G.nx) % G.ny), k = (int)(idx / ((long long)G.nx * G.ny));
    const float x = __fadd_rn(G.ox, __fmul_rn(G.voxel, (float)i));
    const float y = __fadd_rn(G.oy, __fmul_rn(G.voxel, (float)j));
    const float z = __fadd_rn(G.oz, __fmul_rn(G.voxel, (float)k));
    float sdf = S.sdf[idx], r = S.r[idx], g = S.g[idx], b = S.b[idx];
    int w = S.weight[idx], carve = S.carve[idx], cw = S.cw[idx];
    const size_t HW = (size_t)H * W;
    for (int v = 0; v < B; ++v) {
        float pixx, pixy, vz;
        mesh::project(cams + (size_t)v * mesh::kCamStride, H, W, x, y, z, pixx, pixy, vz);
        if (!(vz > kZcull)) continue;
        const float fc = rintf(pixx), fr = rintf(pixy);           // nearest pixel centre, ties to even
        if (!(fc >= 0.f && fc < (float)W && fr >= 0.f && fr < (float)H)) continue;
        const size_t pix = (size_t)fr * W + (size_t)fc;
        const float d = depth[((size_t)v * 2 + 1) * HW + pix];
        if (d == 0.f) {                                          // no surface: alpha < 0.5 along this ray
            ++carve;
            continue;
        }
        const float eta = __fsub_rn(d, vz);
        if (eta < -G.trunc) continue;                            // hidden behind the surface
        const float s = fminf(1.f, __fdiv_rn(eta, G.trunc));
        sdf = __fdiv_rn(__fadd_rn(__fmul_rn(sdf, (float)w), s), (float)(w + 1));
        ++w;
        if (fabsf(eta) < G.trunc) {
            const float a = __fsub_rn(1.f, final_T[(size_t)v * HW + pix]);   // >= 0.5 where the median depth is set
            const float *im = image + (size_t)v * 3 * HW + pix;
            r = __fadd_rn(r, __fdiv_rn(im[0], a));
            g = __fadd_rn(g, __fdiv_rn(im[HW], a));
            b = __fadd_rn(b, __fdiv_rn(im[2 * HW], a));
            ++cw;
        }
    }
    S.sdf[idx] = sdf; S.r[idx] = r; S.g[idx] = g; S.b[idx] = b;
    S.weight[idx] = w; S.carve[idx] = carve; S.cw[idx] = cw;
}

// ---- mesher ---------------------------------------------------------------------------------------------------------------------
// The value the mesher reads at a sample: +1 on the outer layer and where carved at least min_carve times, -1 where no view saw in
// front of it, else the fused sdf.  Inside iff < 0.
__device__ __forceinline__ float sample_value(const Grid &G, const State &S, int i, int j, int k, long long idx, int min_carve)
{
    if (i == 0 || j == 0 || k == 0 || i == G.nx - 1 || j == G.ny - 1 || k == G.nz - 1) return 1.f;
    if (S.carve[idx] >= min_carve) return 1.f;
    if (S.weight[idx] == 0) return -1.f;
    return S.sdf[idx];
}

struct Cube {
    float s[8];
    unsigned present;        // bit c: corner c lies in the grid
    unsigned in;             // bit c: corner c is inside
};

__device__ __forceinline__ long long corner_index(const Grid &G, long long idx, int q)
{
    return idx + (q & 1) + (long long)((q >> 1) & 1) * G.nx + (long long)((q >> 2) & 1) * G.nx * G.ny;
}

__device__ __forceinline__ void load_cube(const Grid &G, const State &S, int i, int j, int k, long long idx, int min_carve, Cube &c)
{
    c.present = 0;
    c.in = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const int dx = q & 1, dy = (q >> 1) & 1, dz = (q >> 2) & 1;
        c.s[q] = 1.f;
        if (i + dx < G.nx && j + dy < G.ny && k + dz < G.nz) {
            c.present |= 1u << q;
            c.s[q] = sample_value(G, S, i + dx, j + dy, k + dz, corner_index(G, idx, q), min_carve);
            if (c.s[q] < 0.f) c.in |= 1u << q;
        }
    }
}

__device__ __forceinline__ unsigned crossing_mask(const Cube &c)
{
    unsigned m = 0;
#pragma unroll
    for (int slot = 0; slot < 7; ++slot) {
        const int q = mask_of_slot(slot);
        if (((c.present >> q) & 1) && (((c.in >> q) ^ c.in) & 1)) m |= 1u << slot;
    }
    return m;
}

__device__ __forceinline__ int tet_case(const Cube &c, int t)
{
    int cs = 0;
#pragma unroll
    for (int v = 0; v < 4; ++v) cs |= ((c.in >> c_table.corner[t][v]) & 1) << v;
    return cs;
}

__global__ void __launch_bounds__(256)
tsdf_count_kernel(Grid G, State S, int min_carve, unsigned char *__restrict__ vmask, int *__restrict__ vcnt, int *__restrict__ fcnt)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx == 0) { vcnt[G.N] = 0; fcnt[G.N] = 0; }
    if (idx >= G.N) return;
    const int i = (int)(idx % G.nx), j = (int)((idx / G.nx) % G.ny), k = (int)(idx / ((long long)G.nx * G.ny));
    Cube c;
    load_cube(G, S, i, j, k, idx, min_carve, c);
    const unsigned m = crossing_mask(c);
    vmask[idx] = (unsigned char)m;
    vcnt[idx] = __popc(m);
    int nt = 0;
    if (c.present == 0xffu)
#pragma unroll
        for (int t = 0; t < 6; ++t) nt += c_table.ntri[t][tet_case(c, t)];
    fcnt[idx] = nt;
}

// mean colour of a sample (0 where no colour was fused)
__device__ __forceinline__ void mean_color(const State &S, long long idx, float out[3], int &cw)
{
    cw = S.cw[idx];
    const float n = (float)cw;
    out[0] = cw ? __fdiv_rn(S.r[idx], n) : 0.f;
    out[1] = cw ? __fdiv_rn(S.g[idx], n) : 0.f;
    out[2] = cw ? __fdiv_rn(S.b[idx], n) : 0.f;
}

__global__ void __launch_bounds__(256)
tsdf_emit_kernel(Grid G, State S, int min_carve, const unsigned char *__restrict__ vmask, const int *__restrict__ voff,
                 const int *__restrict__ foff, long long vcap, long long fcap, float *__restrict__ verts, float *__restrict__ colors,
                 int *__restrict__ faces)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= G.N) return;
    const int i = (int)(idx % G.nx), j = (int)((idx / G.nx) % G.ny), k = (int)(idx / ((long long)G.nx * G.ny));
    Cube c;
    load_cube(G, S, i, j, k, idx, min_carve, c);
    const unsigned m = vmask[idx];
    if (m) {
        float c0[3];
        int cw0;
        mean_color(S, idx, c0, cw0);
        long long v = voff[idx];
#pragma unroll
        for (int slot = 0; slot < 7; ++slot) {
            if (!((m >> slot) & 1)) continue;
            const int q = mask_of_slot(slot);
            const float s0 = c.s[0], s1 = c.s[q];
            const float t = __fdiv_rn(s0, __fsub_rn(s0, s1));
            if (v < vcap) {
                const float g[3] = {__fadd_rn((float)i, __fmul_rn(t, (float)(q & 1))), __fadd_rn((float)j, __fmul_rn(t, (float)((q >> 1) & 1))),
                                    __fadd_rn((float)k, __fmul_rn(t, (float)((q >> 2) & 1)))};
                float *o = verts + 3 * v;
                o[0] = __fadd_rn(G.ox, __fmul_rn(G.voxel, g[0]));
                o[1] = __fadd_rn(G.oy, __fmul_rn(G.voxel, g[1]));
                o[2] = __fadd_rn(G.oz, __fmul_rn(G.voxel, g[2]));
                float c1[3];
                int cw1;
                mean_color(S, corner_index(G, idx, q), c1, cw1);
                float *oc = colors + 3 * v;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const float x0 = cw0 ? c0[a] : c1[a], x1 = cw1 ? c1[a] : c0[a];
                    oc[a] = __fadd_rn(x0, __fmul_rn(t, __fsub_rn(x1, x0)));
                }
            }
            ++v;
        }
    }
    if (c.present != 0xffu) return;
    long long f = foff[idx];
    if (f == foff[idx + 1]) return;
    for (int t = 0; t < 6; ++t) {
        const int cs = tet_case(c, t);
        const int nt = c_table.ntri[t][cs];
        for (int n = 0; n < nt; ++n, ++f) {
            if (f >= fcap) continue;
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const int e = c_table.edge[t][cs][3 * n + q];
                const long long own = corner_index(G, idx, c_table.owner[t][e]);
                const int slot = c_table.slot[t][e];
                faces[3 * f + q] = voff[own] + __popc((unsigned)vmask[own] & ((1u << slot) - 1u));
            }
        }
    }
}

int check_grid(const GaTsdfDesc *d, const char *fn, Grid &G)
{
    GA_REQUIRE(d, "%s: NULL grid descriptor", fn);
    GA_REQUIRE(d->nx >= kMinSide && d->nx <= kMaxSide && d->ny >= kMinSide && d->ny <= kMaxSide && d->nz >= kMinSide && d->nz <= kMaxSide,
               "%s: grid %d x %d x %d outside [%d, %d]^3", fn, d->nx, d->ny, d->nz, kMinSide, kMaxSide);
    GA_REQUIRE(isfinite(d->voxel) && d->voxel > 0.f, "%s: voxel size %g must be finite and > 0", fn, (double)d->voxel);
    GA_REQUIRE(isfinite(d->trunc) && d->trunc > 0.f, "%s: truncation %g must be finite and > 0", fn, (double)d->trunc);
    GA_REQUIRE(isfinite(d->origin[0]) && isfinite(d->origin[1]) && isfinite(d->origin[2]), "%s: origin must be finite", fn);
    G = Grid{d->nx, d->ny, d->nz, (long long)d->nx * d->ny * d->nz, d->origin[0], d->origin[1], d->origin[2], d->voxel, d->trunc};
    return GA_OK;
}

struct MeshWs {
    unsigned char *vmask;
    int *vcnt, *fcnt;
    void *temp;
    size_t temp_bytes, total;
};

MeshWs carve_ws(void *p, long long N)
{
    size_t temp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, temp, (int *)nullptr, (int *)nullptr, (int)(N + 1));
    Carver c(p);
    MeshWs w;
    w.vmask = c.take<unsigned char>((size_t)N);
    w.vcnt = c.take<int>((size_t)N + 1);
    w.fcnt = c.take<int>((size_t)N + 1);
    w.temp = c.take<unsigned char>(temp);
    w.temp_bytes = temp;
    w.total = c.used();
    return w;
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" size_t ga_tsdf_state_bytes(const GaTsdfDesc *d)
{
    Grid G;
    if (check_grid(d, "ga_tsdf_state_bytes", G) != GA_OK) return 0;
    return (size_t)kPlanes * 4 * (size_t)G.N;
}

extern "C" int ga_tsdf_reset(const GaTsdfDesc *d, void *state, void *stream)
{
    Grid G;
    const int rc = check_grid(d, "ga_tsdf_reset", G);
    if (rc != GA_OK) return rc;
    GA_REQUIRE(state, "ga_tsdf_reset: state is NULL");
    GA_CHECK_CUDA(cudaMemsetAsync(state, 0, (size_t)kPlanes * 4 * (size_t)G.N, static_cast<cudaStream_t>(stream)));
    return GA_OK;
}

extern "C" int ga_tsdf_integrate(const GaTsdfDesc *d, int32_t B, int32_t H, int32_t W, const float *cams, const float *depth,
                                 const float *image, const float *final_T, void *state, void *stream_)
{
    Grid G;
    const int rc = check_grid(d, "ga_tsdf_integrate", G);
    if (rc != GA_OK) return rc;
    GA_REQUIRE(B >= 1 && B <= kMaxViews, "ga_tsdf_integrate: %d views outside [1, %d]", B, kMaxViews);
    GA_REQUIRE(H >= 1 && H <= kMaxImageSide && W >= 1 && W <= kMaxImageSide, "ga_tsdf_integrate: image %d x %d outside [1, %d]^2", H, W,
               kMaxImageSide);
    GA_REQUIRE(cams && depth && image && final_T && state, "ga_tsdf_integrate: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("tsdf_integrate_kernel", stream);
      tsdf_integrate_kernel<<<cdiv(G.N, 256), 256, 0, stream>>>(G, B, H, W, cams, depth, image, final_T, state_of(state, G.N)); }
    GA_CHECK_LAUNCH("tsdf_integrate_kernel");
    return GA_OK;
}

extern "C" size_t ga_tsdf_mesh_workspace_bytes(const GaTsdfDesc *d)
{
    Grid G;
    if (check_grid(d, "ga_tsdf_mesh_workspace_bytes", G) != GA_OK) return 0;
    return carve_ws(nullptr, G.N).total;
}

extern "C" int ga_tsdf_mesh_count(const GaTsdfDesc *d, const void *state, int32_t min_carve, void *workspace, size_t workspace_bytes,
                                  int32_t *totals, void *stream_)
{
    Grid G;
    const int rc = check_grid(d, "ga_tsdf_mesh_count", G);
    if (rc != GA_OK) return rc;
    GA_REQUIRE(min_carve >= 1, "ga_tsdf_mesh_count: min_carve %d must be >= 1", min_carve);
    GA_REQUIRE(state && workspace && totals, "ga_tsdf_mesh_count: NULL pointer argument");
    const MeshWs w = carve_ws(workspace, G.N);
    if (workspace_bytes < w.total) {
        set_error("ga_tsdf_mesh_count: workspace of %zu bytes, %zu needed", workspace_bytes, w.total);
        return GA_ERR_CAPACITY;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const State S = state_of(const_cast<void *>(state), G.N);
    { ProfScope _ps("tsdf_count_kernel", stream);
      tsdf_count_kernel<<<cdiv(G.N, 256), 256, 0, stream>>>(G, S, min_carve, w.vmask, w.vcnt, w.fcnt); }
    GA_CHECK_LAUNCH("tsdf_count_kernel");
    size_t tb = w.temp_bytes;
    { ProfScope _ps("tsdf_scan", stream);
      GA_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.vcnt, w.vcnt, (int)(G.N + 1), stream));
      GA_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.fcnt, w.fcnt, (int)(G.N + 1), stream)); }
    count_launch(2);
    GA_CHECK_CUDA(cudaMemcpyAsync(totals, w.vcnt + G.N, sizeof(int), cudaMemcpyDeviceToDevice, stream));
    GA_CHECK_CUDA(cudaMemcpyAsync(totals + 1, w.fcnt + G.N, sizeof(int), cudaMemcpyDeviceToDevice, stream));
    return GA_OK;
}

extern "C" int ga_tsdf_mesh_emit(const GaTsdfDesc *d, const void *state, int32_t min_carve, const void *workspace, size_t workspace_bytes,
                                 int64_t vertex_capacity, int64_t face_capacity, float *verts, float *colors, int32_t *faces, void *stream_)
{
    Grid G;
    const int rc = check_grid(d, "ga_tsdf_mesh_emit", G);
    if (rc != GA_OK) return rc;
    GA_REQUIRE(min_carve >= 1, "ga_tsdf_mesh_emit: min_carve %d must be >= 1", min_carve);
    GA_REQUIRE(vertex_capacity >= 0 && face_capacity >= 0, "ga_tsdf_mesh_emit: negative capacity");
    GA_REQUIRE(state && workspace && (vertex_capacity == 0 || (verts && colors)) && (face_capacity == 0 || faces),
               "ga_tsdf_mesh_emit: NULL pointer argument");
    const MeshWs w = carve_ws(const_cast<void *>(workspace), G.N);
    if (workspace_bytes < w.total) {
        set_error("ga_tsdf_mesh_emit: workspace of %zu bytes, %zu needed", workspace_bytes, w.total);
        return GA_ERR_CAPACITY;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const State S = state_of(const_cast<void *>(state), G.N);
    { ProfScope _ps("tsdf_emit_kernel", stream);
      tsdf_emit_kernel<<<cdiv(G.N, 256), 256, 0, stream>>>(G, S, min_carve, w.vmask, w.vcnt, w.fcnt, vertex_capacity, face_capacity, verts,
                                                          colors, faces); }
    GA_CHECK_LAUNCH("tsdf_emit_kernel");
    return GA_OK;
}
