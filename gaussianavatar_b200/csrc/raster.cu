// Differentiable 3D-Gaussian tile rasterizer for sm_90a — forward (K1..K6) and backward (K7, fused K8/K9), for one frame or
// for all frames of a training step in one set of launches.
//
// Replaces what the reference reaches through `GaussianRasterizer(raster_settings)(...)`
// (/root/reference gaussian_renderer/__init__.py:36-48; [UPSTREAM] diff-gaussian-rasterization, not vendored).
// Algorithm and constants: SURVEY.md §8 "a-8 forward spec" / "a-9 backward spec".  Written from that specification,
// not from upstream source.  The RESULTS are upstream's (tile ranges, depth-ordered per-tile lists, image, gradients);
// the way they are produced is not:
//
//   binning   upstream: duplicateWithKeys -> global 64-bit radix sort of all (tile | depth) keys -> identifyTileRanges, with a
//             device->host read of the instance count in the middle.  Here: K1 counts instances per tile, ONE CTA scans the
//             counts (tile ranges fall out directly), K3 scatters (depth bits | Gaussian index) into the tile's bucket and one
//             CTA per tile sorts its bucket in shared memory.  The order inside a tile is upstream's (depth bits, then Gaussian
//             index = the stable order of its key sort), no launch shape depends on the instance count, and nothing is read back
//             by the host: the binning buffer has a caller-chosen capacity, an overflow raises a device-side flag
//             (status[1]) and the affected tiles are skipped, never overrun.
//   K6        one warp per 8x4-pixel sub-tile walks the tile list on its own (no CTA barriers): 32 entries are tested against
//             the sub-tile in parallel and only the survivors are composited.  The sort kernel leaves packed per-instance
//             records (centre, conic, opacity, colour, cull radius) in list order, so the walk streams instead of gathering.
//             Every 256 list positions each pixel's (T, C) is checkpointed ...
//   K7        ... so that the backward runs ONE CTA PER 256-ENTRY SEGMENT of a tile list, all segments in parallel, each
//             starting from the checkpoint behind it (upstream replays a whole tile list serially in one CTA).
//
// Arithmetic contract (DESIGN.md §3): every value that feeds an INTEGER decision (depth key bits, radius, tile rect)
// is computed with explicit round-to-nearest intrinsics in exactly the operation order of oracle/raster_oracle_impl.inc,
// so radii / ranges / list order are bit-exact against the CPU oracle regardless of nvcc's FMA contraction.
#include <cub/cub.cuh>

#include <type_traits>

#include "common.cuh"

namespace ga {
namespace {

constexpr int kTile = 16;
constexpr int kBlock = kTile * kTile;
constexpr int kSeg = 256;            // list positions per checkpoint interval = per backward work item
constexpr int kSortThreads = 512;
constexpr int kSortMax = 8192;       // keys one CTA sorts in shared memory at a time (64 KB): long tile lists (>= kSortSmallMax keys)
constexpr int kSortSmallThreads = 128;
constexpr int kSortSmallMax = 2048;  // short tile lists go to 128-thread CTAs (16 KB of keys, a dozen CTAs per SM): with 512 threads a
                                     // 500-entry bucket is mostly barrier waits (barrier stall 25 per issue in ncu, 19 % issue-active)
constexpr int kStatusInts = 16;      // status[0] instances, [1] overflow flag, [2] segments, [3] non-empty tiles, [4+b] first instance of
                                     // frame b (b <= 8), [13] tiles with >= kSortSmallMax entries, [15] the caller's serial number

struct Dims {
    int B, P, H, W, gx, gy, T;
};
inline Dims make_dims(int B, int P, int H, int W)
{
    Dims d{B, P, H, W, cdiv(W, kTile), cdiv(H, kTile), 0};
    d.T = d.gx * d.gy;
    return d;
}

struct GeomViews {
    float *depth;
    float2 *xy;
    float4 *conic_o;
    float *cov3d;
    uint32_t *tiles;
    ushort4 *rect;
    size_t total;
};

GeomViews carve_geom(void *buf, size_t BP)
{
    Carver c(buf);
    GeomViews g;
    const size_t n = BP > 0 ? BP : 1;
    g.depth = c.take<float>(n);
    g.xy = c.take<float2>(n);
    g.conic_o = c.take<float4>(n);
    g.cov3d = c.take<float>(6 * n);
    g.tiles = c.take<uint32_t>(n);
    g.rect = c.take<ushort4>(n);
    g.total = c.used();
    return g;
}

struct ImgViews {
    float *final_T;          // [B][H*W]
    uint32_t *n_contrib;     // [B][H*W]
    float4 *final_state;     // [B*T][256] tile-major (T, C0, C1, C2 without background)
    uint2 *ranges;           // [B*T] global [start, end) into the instance arrays
    uint32_t *count;         // [B*T] instances per tile (K1)
    uint32_t *cursor;        // [B*T] scatter cursor (starts at ranges.x)
    uint32_t *seg_start;     // [B*T+1] exclusive scan of ceil(count/256)
    uint32_t *tile_maxc;     // [B*T] max n_contrib of the tile's pixels
    uint32_t *order;         // [B*T] tiles by decreasing list length (classes of log2), empty tiles last
    int32_t *status;         // [kStatusInts]
    size_t total;
};

ImgViews carve_img(void *buf, const Dims &d)
{
    Carver c(buf);
    ImgViews v;
    const size_t hw = (size_t)d.B * d.H * d.W, BT = (size_t)d.B * d.T;
    v.final_T = c.take<float>(hw ? hw : 1);
    v.n_contrib = c.take<uint32_t>(hw ? hw : 1);
    v.final_state = c.take<float4>((BT ? BT : 1) * kBlock);
    v.ranges = c.take<uint2>(BT ? BT : 1);
    v.count = c.take<uint32_t>(BT ? BT : 1);
    v.cursor = c.take<uint32_t>(BT ? BT : 1);
    v.seg_start = c.take<uint32_t>(BT + 1);
    v.tile_maxc = c.take<uint32_t>(BT ? BT : 1);
    v.order = c.take<uint32_t>(BT ? BT : 1);
    v.status = c.take<int32_t>(kStatusInts);
    v.total = c.used();
    return v;
}

struct BinViews {
    uint64_t *bucket;        // [cap] (depth bits << 32 | Gaussian index), grouped by tile, unsorted inside a tile
    uint32_t *point_list;    // [cap] Gaussian index in upstream's sorted order
    float4 *recA, *recB, *recC;   // [cap] packed records in list order: (x, y, cull r^2, idx) (conic xyz, opacity) (r, g, b, z)
                                  // (z: the view depth when the forward writes depth, else 0)
    float4 *ckpt;            // [max_segments][256] per-pixel (T, C) at the start of each 256-entry segment
    uint32_t *seg_tile;      // [max_segments] segment -> tile
    size_t max_segments;
    size_t total;
};

inline size_t max_segments_for(int64_t cap, const Dims &d) { return (size_t)(cap / kSeg) + (size_t)d.B * d.T + 1; }

BinViews carve_bin(void *buf, int64_t cap, const Dims &d)
{
    Carver c(buf);
    BinViews b;
    const size_t n = cap > 0 ? (size_t)cap : 1;
    b.max_segments = max_segments_for(cap, d);
    b.bucket = c.take<uint64_t>(n);
    b.point_list = c.take<uint32_t>(n);
    b.recA = c.take<float4>(n);
    b.recB = c.take<float4>(n);
    b.recC = c.take<float4>(n);
    b.ckpt = c.take<float4>(b.max_segments * kBlock);
    b.seg_tile = c.take<uint32_t>(b.max_segments);
    b.total = c.used();
    return b;
}

// The depth state the training forward with depth leaves for the depth backward: each pixel's D = sum w z at the start of every
// 256-entry segment (laid out as BinViews::ckpt) and at the end of its list (laid out as ImgViews::final_state).
struct DepthState {
    float *ckpt;             // [max_segments][256]
    float *final;            // [B*T][256] tile-major
    size_t total;
};

DepthState carve_dstate(void *buf, int64_t cap, const Dims &d)
{
    Carver c(buf);
    DepthState s;
    const size_t BT = (size_t)d.B * d.T;
    s.ckpt = c.take<float>(max_segments_for(cap, d) * kBlock);
    s.final = c.take<float>((BT ? BT : 1) * kBlock);
    s.total = c.used();
    return s;
}

// ---- contraction-proof arithmetic (mirrors oracle/raster_oracle_impl.inc op for op) ----
__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fma_(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }

__device__ __forceinline__ float xf_row(const float *__restrict__ M, int r, float x, float y, float z)
{
    float t = mul_(M[r], x);
    t = fma_(M[4 + r], y, t);
    t = fma_(M[8 + r], z, t);
    return add_(t, M[12 + r]);
}

struct Cov3 {
    float v[6];
};

__device__ __forceinline__ void quat_to_rot(float qr, float qx, float qy, float qz, float R[3][3])
{
    R[0][0] = sub_(1.f, mul_(2.f, add_(mul_(qy, qy), mul_(qz, qz))));
    R[0][1] = mul_(2.f, sub_(mul_(qx, qy), mul_(qr, qz)));
    R[0][2] = mul_(2.f, add_(mul_(qx, qz), mul_(qr, qy)));
    R[1][0] = mul_(2.f, add_(mul_(qx, qy), mul_(qr, qz)));
    R[1][1] = sub_(1.f, mul_(2.f, add_(mul_(qx, qx), mul_(qz, qz))));
    R[1][2] = mul_(2.f, sub_(mul_(qy, qz), mul_(qr, qx)));
    R[2][0] = mul_(2.f, sub_(mul_(qx, qz), mul_(qr, qy)));
    R[2][1] = mul_(2.f, add_(mul_(qy, qz), mul_(qr, qx)));
    R[2][2] = sub_(1.f, mul_(2.f, add_(mul_(qx, qx), mul_(qy, qy))));
}

// Where a frame's camera comes from: a device array of kCamStride floats per frame (batched path: view 0..15, proj 16..31,
// tanfovx 32, tanfovy 33, camera centre 34..36, read only by the composite forward) or two device matrices plus host scalars
// (per-frame API, stride 0).
constexpr int kCamStride = 40;
constexpr int kCamPos = 34;
struct CamSrc {
    const float *view, *proj, *tan;
    int stride;
    float tanx, tany;
};

// Colour and covariance sources of the per-frame API beyond precomputed colours + scale / rotation (GaRasterColorCov): spherical-
// harmonic colours evaluated in K1 (kSH) and precomputed 3D covariances (kCov).  The batched path passes it zeroed.
struct ColorCov {
    const float *shs;        // [P, M, 3] coefficient-major RGB triples
    int D, M;                // active degree 0..3, coefficients per Gaussian
    bool vec4;               // every row starts 16-byte aligned (M % 4 == 0, aligned base): whole-sector float4 accesses
    const float *campos;     // [3]
    const float *cov3D;      // [P, 6] (xx, xy, xz, yy, yz, zz)
    float *rgb;              // [P, 3] evaluated colour (K1 writes, K4 packs it)
    uint8_t *clamped;        // [P] bit c: channel c was clamped at 0
    const float *d_rgb;      // [P, 3] dL/drgb accumulated by K7 (backward)
    float *d_sh;             // [P, M, 3]
    float *d_cov3D;          // [P, 6]
};

constexpr float kShC0 = 0.28209479177387814f, kShC1 = 0.4886025119029199f;
constexpr float kShC2_0 = 1.0925484305920792f, kShC2_1 = -1.0925484305920792f, kShC2_2 = 0.31539156525252005f,
                kShC2_3 = -1.0925484305920792f, kShC2_4 = 0.5462742152960396f;
constexpr float kShC3_0 = -0.5900435899266435f, kShC3_1 = 2.890611442640554f, kShC3_2 = -0.4570457994644658f,
                kShC3_3 = 0.3731763325901154f, kShC3_4 = -0.4570457994644658f, kShC3_5 = 1.445305721320277f,
                kShC3_6 = -0.5900435899266435f;

// The 16 real SH basis functions up to degree 3 at the unit direction (x, y, z).
__device__ __forceinline__ void sh_basis(float x, float y, float z, float b[16])
{
    const float xx = x * x, yy = y * y, zz = z * z;
    b[0] = kShC0;
    b[1] = -kShC1 * y; b[2] = kShC1 * z; b[3] = -kShC1 * x;
    b[4] = kShC2_0 * x * y; b[5] = kShC2_1 * y * z; b[6] = kShC2_2 * (2.f * zz - xx - yy); b[7] = kShC2_3 * x * z;
    b[8] = kShC2_4 * (xx - yy);
    b[9] = kShC3_0 * y * (3.f * xx - yy); b[10] = kShC3_1 * x * y * z; b[11] = kShC3_2 * y * (4.f * zz - xx - yy);
    b[12] = kShC3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy); b[13] = kShC3_4 * x * (4.f * zz - xx - yy);
    b[14] = kShC3_5 * z * (xx - yy); b[15] = kShC3_6 * x * (xx - 3.f * yy);
}

// Visits the first n (<= 48) floats of one Gaussian's SH row as f(e, value), e compile-time after unrolling.  With vec4 the row is
// read in float4s, so a warp's loads use whole 32-byte sectors although its lanes' rows lie 12*M bytes apart.
template <class F>
__device__ __forceinline__ void sh_row_load(const float *__restrict__ row, int n, bool vec4, F f)
{
    if (vec4) {
#pragma unroll
        for (int q = 0; q < 12; ++q)
            if (4 * q < n) {
                const float4 v = __ldg(reinterpret_cast<const float4 *>(row) + q);
                f(4 * q, v.x); f(4 * q + 1, v.y); f(4 * q + 2, v.z); f(4 * q + 3, v.w);
            }
    } else {
#pragma unroll
        for (int e = 0; e < 48; ++e)
            if (e < n) f(e, __ldg(row + e));
    }
}

// Writes a whole SH row of nrow = 3*M floats: f(e) for e < 48 (compile-time after unrolling), 0 beyond.
template <class F>
__device__ __forceinline__ void sh_row_store(float *__restrict__ row, int nrow, bool vec4, F f)
{
    if (vec4) {
        float4 *r4 = reinterpret_cast<float4 *>(row);
#pragma unroll
        for (int q = 0; q < 12; ++q)
            if (4 * q < nrow) r4[q] = make_float4(f(4 * q), f(4 * q + 1), f(4 * q + 2), f(4 * q + 3));
        for (int q = 12; 4 * q < nrow; ++q) r4[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
#pragma unroll
        for (int e = 0; e < 48; ++e)
            if (e < nrow) row[e] = f(e);
        for (int e = 48; e < nrow; ++e) row[e] = 0.f;
    }
}

// The SH colour of one Gaussian's row of degree D seen from campos: r = max(sum_k basis_k(dir) sh_k + 0.5, 0) with
// dir = (mean - campos) / |mean - campos|; r must come in zeroed.  Returns the clamp bits (bit c: channel c was clamped at 0).
__device__ __forceinline__ uint32_t sh_eval(const float *__restrict__ row, int D, bool vec4, const float *__restrict__ campos, float px,
                                            float py, float pz, float r[3])
{
    uint32_t cl = 0;
    const float vx = px - __ldg(campos), vy = py - __ldg(campos + 1), vz = pz - __ldg(campos + 2);
    const float inv = 1.f / sqrtf(vx * vx + vy * vy + vz * vz);
    float b[16];
    sh_basis(vx * inv, vy * inv, vz * inv, b);
    const int n = 3 * (D + 1) * (D + 1);
    sh_row_load(row, n, vec4, [&](int e, float v) { if (e < n) r[e % 3] += b[e / 3] * v; });
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        r[ch] += 0.5f;
        if (r[ch] < 0.f) { cl |= 1u << ch; r[ch] = 0.f; }
    }
    return cl;
}

// K1's SH colour of Gaussian i (sh_eval from cc.campos).  Culled Gaussians (live = false) get rgb 0 and no clamp bits; ordinary fp32,
// no integer decision depends on it.
__device__ __forceinline__ void sh_color_fwd(const ColorCov &cc, size_t i, float px, float py, float pz, bool live)
{
    float r[3] = {0.f, 0.f, 0.f};
    uint32_t cl = 0;
    if (live) cl = sh_eval(cc.shs + i * 3 * cc.M, cc.D, cc.vec4, cc.campos, px, py, pz, r);
    cc.rgb[3 * i] = r[0]; cc.rgb[3 * i + 1] = r[1]; cc.rgb[3 * i + 2] = r[2];
    cc.clamped[i] = (uint8_t)cl;
}

// The static set of the composite forward (GaRasterScene): Ps Gaussians shared by every frame (read with frame stride 0) that
// follow each frame's P dynamic ones in its index space.  K1 evaluates their SH colours for each frame's camera centre into rgb.
struct SceneSet {
    const float *means3D, *scales, *rotations, *opacities, *shs;   // [Ps,3] [Ps,3] [Ps,4] [Ps] [Ps,M,3]
    int Ps, D, M;
    bool vec4;               // as ColorCov::vec4
    float *rgb;              // [B, Ps, 3]
};

// Backward of sh_color_fwd for a visible Gaussian: writes the whole d_sh row (basis_k * dL/drgb, 0 on clamped channels and for
// k >= (D+1)^2) and adds the direction term, pushed through the normalisation, to dmean.
__device__ __forceinline__ void sh_color_bwd(const ColorCov &cc, size_t i, float px, float py, float pz, float dmean[3])
{
    const uint32_t cl = cc.clamped[i];
    float g[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) g[ch] = (cl >> ch) & 1u ? 0.f : cc.d_rgb[3 * i + ch];
    const float vx = px - __ldg(cc.campos), vy = py - __ldg(cc.campos + 1), vz = pz - __ldg(cc.campos + 2);
    const float inv = 1.f / sqrtf(vx * vx + vy * vy + vz * vz);
    const float x = vx * inv, y = vy * inv, z = vz * inv;
    float b[16];
    sh_basis(x, y, z, b);
    const int n = 3 * (cc.D + 1) * (cc.D + 1);
    float s[16];                     // s_k = sh_k . dL/drgb
#pragma unroll
    for (int k = 0; k < 16; ++k) s[k] = 0.f;
    sh_row_load(cc.shs + i * 3 * cc.M, n, cc.vec4, [&](int e, float v) { if (e < n) s[e / 3] += v * g[e % 3]; });
    sh_row_store(cc.d_sh + i * 3 * cc.M, 3 * cc.M, cc.vec4, [&](int e) { return e < n ? b[e / 3] * g[e % 3] : 0.f; });
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    const float ddx = -kShC1 * s[3] + kShC2_0 * y * s[4] - 2.f * kShC2_2 * x * s[6] + kShC2_3 * z * s[7] + 2.f * kShC2_4 * x * s[8] +
                      6.f * kShC3_0 * xy * s[9] + kShC3_1 * yz * s[10] - 2.f * kShC3_2 * xy * s[11] - 6.f * kShC3_3 * xz * s[12] +
                      kShC3_4 * (4.f * zz - 3.f * xx - yy) * s[13] + 2.f * kShC3_5 * xz * s[14] + 3.f * kShC3_6 * (xx - yy) * s[15];
    const float ddy = -kShC1 * s[1] + kShC2_0 * x * s[4] + kShC2_1 * z * s[5] - 2.f * kShC2_2 * y * s[6] - 2.f * kShC2_4 * y * s[8] +
                      3.f * kShC3_0 * (xx - yy) * s[9] + kShC3_1 * xz * s[10] + kShC3_2 * (4.f * zz - xx - 3.f * yy) * s[11] -
                      6.f * kShC3_3 * yz * s[12] - 2.f * kShC3_4 * xy * s[13] - 2.f * kShC3_5 * yz * s[14] - 6.f * kShC3_6 * xy * s[15];
    const float ddz = kShC1 * s[2] + kShC2_1 * y * s[5] + 4.f * kShC2_2 * z * s[6] + kShC2_3 * x * s[7] + kShC3_1 * xy * s[10] +
                      8.f * kShC3_2 * yz * s[11] + kShC3_3 * (6.f * zz - 3.f * xx - 3.f * yy) * s[12] + 8.f * kShC3_4 * xz * s[13] +
                      kShC3_5 * (xx - yy) * s[14];
    // d dir / d mean = (I - dir dir^T) / |v|
    const float dot = x * ddx + y * ddy + z * ddz;
    dmean[0] += (ddx - x * dot) * inv;
    dmean[1] += (ddy - y * dot) * inv;
    dmean[2] += (ddz - z * dot) * inv;
}

// Per-Gaussian part of K1; returns the tile rect (zero area if the Gaussian is culled).  kCov: Sigma is read from cov_pre (this
// Gaussian's six values) instead of being built from scales / rotations / mod; everything after Sigma is the same op sequence.
// kAA (upstream's `antialiasing`): the stored opacity is o rho, rho = sqrt(max(2.5e-5, det(Sigma2) / det(Sigma2 + 0.3 I))) with
// Sigma2 the projected covariance before the dilation; every other output is the call without it's, bit for bit.
// i indexes the outputs, src the rows of means3D / scales.
template <bool kCov, bool kAA = false>
__device__ __forceinline__ ushort4
preprocess_one(int il, size_t i, size_t src, int H, int W, int gx, int gy, const float *view, const float *proj, float tanfovx, float tanfovy,
               float mod, const float *__restrict__ means3D, const float *__restrict__ scales, const float *__restrict__ rq,
               const float *__restrict__ cov_pre, float opacity, float *__restrict__ depth, float2 *__restrict__ xy,
               float4 *__restrict__ conic_o, float *__restrict__ cov3d, uint32_t *__restrict__ tiles, ushort4 *__restrict__ rect,
               int32_t *__restrict__ radii)
{
    const ushort4 none = make_ushort4(0, 0, 0, 0);
    radii[i] = 0;
    tiles[i] = 0;
    depth[i] = 0.f;
    xy[i] = make_float2(0.f, 0.f);
    conic_o[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    rect[i] = make_ushort4(0, 0, 0, 0);
#pragma unroll
    for (int k = 0; k < 6; ++k) cov3d[6 * (size_t)i + k] = 0.f;

    const float px = means3D[3 * src], py = means3D[3 * src + 1], pz = means3D[3 * src + 2];
    const float tvx = xf_row(view, 0, px, py, pz), tvy = xf_row(view, 1, px, py, pz), tvz = xf_row(view, 2, px, py, pz);
    if (tvz <= 0.2f) return none;

    const float hx = xf_row(proj, 0, px, py, pz), hy = xf_row(proj, 1, px, py, pz), hw = xf_row(proj, 3, px, py, pz);
    const float p_w = div_(1.f, add_(hw, 0.0000001f));
    const float ndc_x = mul_(hx, p_w), ndc_y = mul_(hy, p_w);

    float S00, S01, S02, S11, S12, S22;
    if constexpr (kCov) {
        S00 = cov_pre[0]; S01 = cov_pre[1]; S02 = cov_pre[2]; S11 = cov_pre[3]; S12 = cov_pre[4]; S22 = cov_pre[5];
    } else {
        const float sv[3] = {mul_(mod, scales[3 * src]), mul_(mod, scales[3 * src + 1]), mul_(mod, scales[3 * src + 2])};
        float Rm[3][3];
        quat_to_rot(rq[0], rq[1], rq[2], rq[3], Rm);
        float Mm[3][3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int k = 0; k < 3; ++k) Mm[a][k] = mul_(sv[a], Rm[k][a]);
        float Sg[3][3];
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int k = j; k < 3; ++k) {
                float t = mul_(Mm[0][j], Mm[0][k]);
                t = fma_(Mm[1][j], Mm[1][k], t);
                t = fma_(Mm[2][j], Mm[2][k], t);
                Sg[j][k] = t;
            }
        S00 = Sg[0][0]; S01 = Sg[0][1]; S02 = Sg[0][2]; S11 = Sg[1][1]; S12 = Sg[1][2]; S22 = Sg[2][2];
    }

    const float focal_x = div_((float)W, mul_(2.f, tanfovx)), focal_y = div_((float)H, mul_(2.f, tanfovy));
    const float limx = mul_(1.3f, tanfovx), limy = mul_(1.3f, tanfovy);
    const float txtz = div_(tvx, tvz), tytz = div_(tvy, tvz);
    const float tx = mul_(fminf(limx, fmaxf(-limx, txtz)), tvz);
    const float ty = mul_(fminf(limy, fmaxf(-limy, tytz)), tvz);
    const float tz2 = mul_(tvz, tvz);
    const float J00 = div_(focal_x, tvz), J02 = div_(-mul_(focal_x, tx), tz2);
    const float J11 = div_(focal_y, tvz), J12 = div_(-mul_(focal_y, ty), tz2);
    float m0[3], m1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        m0[k] = fma_(view[k * 4 + 2], J02, mul_(view[k * 4 + 0], J00));
        m1[k] = fma_(view[k * 4 + 2], J12, mul_(view[k * 4 + 1], J11));
    }
    const float v00 = fma_(S02, m0[2], fma_(S01, m0[1], mul_(S00, m0[0])));
    const float v01 = fma_(S12, m0[2], fma_(S11, m0[1], mul_(S01, m0[0])));
    const float v02 = fma_(S22, m0[2], fma_(S12, m0[1], mul_(S02, m0[0])));
    const float v10 = fma_(S02, m1[2], fma_(S01, m1[1], mul_(S00, m1[0])));
    const float v11 = fma_(S12, m1[2], fma_(S11, m1[1], mul_(S01, m1[0])));
    const float v12 = fma_(S22, m1[2], fma_(S12, m1[1], mul_(S02, m1[0])));
    const float ca0 = fma_(m0[2], v02, fma_(m0[1], v01, mul_(m0[0], v00)));
    const float cb = fma_(m0[2], v12, fma_(m0[1], v11, mul_(m0[0], v10)));
    const float cc0 = fma_(m1[2], v12, fma_(m1[1], v11, mul_(m1[0], v10)));
    const float ca = add_(ca0, 0.3f), cc = add_(cc0, 0.3f);

    const float det = sub_(mul_(ca, cc), mul_(cb, cb));
    if (det == 0.f) return none;
    const float det_inv = div_(1.f, det);
    const float conx = mul_(cc, det_inv), cony = mul_(-cb, det_inv), conz = mul_(ca, det_inv);
    const float mid = mul_(0.5f, add_(ca, cc));
    const float sq = __fsqrt_rn(fmaxf(0.1f, sub_(mul_(mid, mid), det)));
    const float lambda1 = add_(mid, sq), lambda2 = sub_(mid, sq);
    const int radius = (int)ceilf(mul_(3.f, __fsqrt_rn(fmaxf(lambda1, lambda2))));

    const float pixx = (float)__dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)ndc_x, 1.0), (double)W), -1.0), 0.5);
    const float pixy = (float)__dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)ndc_y, 1.0), (double)H), -1.0), 0.5);

    const float rf = (float)radius;
    int rminx = __float2int_rz(div_(sub_(pixx, rf), 16.f)); rminx = min(gx, max(0, rminx));
    int rminy = __float2int_rz(div_(sub_(pixy, rf), 16.f)); rminy = min(gy, max(0, rminy));
    int rmaxx = __float2int_rz(div_(add_(add_(pixx, rf), 15.f), 16.f)); rmaxx = min(gx, max(0, rmaxx));
    int rmaxy = __float2int_rz(div_(add_(add_(pixy, rf), 15.f), 16.f)); rmaxy = min(gy, max(0, rmaxy));
    const int area = (rmaxx - rminx) * (rmaxy - rminy);
    if (area == 0) return none;

    float *c3 = cov3d + 6 * (size_t)i;
    c3[0] = S00; c3[1] = S01; c3[2] = S02; c3[3] = S11; c3[4] = S12; c3[5] = S22;
    depth[i] = tvz;
    radii[i] = radius;
    xy[i] = make_float2(pixx, pixy);
    float o = opacity;
    if constexpr (kAA) {
        const float det0 = sub_(mul_(ca0, cc0), mul_(cb, cb));
        o = mul_(opacity, __fsqrt_rn(fmaxf(2.5e-5f, div_(det0, det))));
    }
    conic_o[i] = make_float4(conx, cony, conz, o);
    tiles[i] = (uint32_t)area;
    const ushort4 rc = make_ushort4((unsigned short)rminx, (unsigned short)rminy, (unsigned short)rmaxx, (unsigned short)rmaxy);
    rect[i] = rc;
    return rc;
}

// Visit every tile of every lane's rect with op(tile, payload-of-the-owning-lane), load-balanced inside the warp: a Gaussian that
// touches a few tiles (the rule) is handled by its own lane; one that touches many (large radius: a serial loop of dependent atomics
// that used to set the kernel's duration) is spread over the 32 lanes, 32 tiles per step.
template <class Op>
__device__ __forceinline__ void for_each_tile_balanced(const ushort4 rc, int gx, uint64_t payload, Op op)
{
    constexpr int kSmall = 4;
    const int lane = threadIdx.x & 31;
    const int w = (int)rc.z - (int)rc.x, area = w * ((int)rc.w - (int)rc.y);
    if (area <= kSmall)
        for (int k = 0; k < area; ++k) op((uint32_t)(((int)rc.y + k / w) * gx + (int)rc.x + k % w), payload);
    uint32_t big = __ballot_sync(0xffffffffu, area > kSmall);
    while (big) {
        const int src = __ffs(big) - 1;
        big &= big - 1;
        const int x0 = __shfl_sync(0xffffffffu, (int)rc.x, src), y0 = __shfl_sync(0xffffffffu, (int)rc.y, src);
        const int ws = __shfl_sync(0xffffffffu, w, src), as = __shfl_sync(0xffffffffu, area, src);
        const uint64_t pl = __shfl_sync(0xffffffffu, payload, src);
        for (int k = lane; k < as; k += 32) op((uint32_t)((y0 + k / ws) * gx + x0 + k % ws), pl);
    }
}

// CTA-local tile table of K1 / K3: an open-addressing hash (tile id -> count / cursor) in shared memory.  A CTA's 256 Gaussians touch
// at most a few thousand distinct tiles wherever they lie on screen, so the table is small (kTileSlots), independent of the image
// size and of how the Gaussians are ordered; an instance whose probe sequence is full (huge Gaussians) falls back to the global
// atomic, consistently in every pass (slots are never freed, so the same probes fail again).
constexpr int kTileSlots = 4096;
constexpr uint32_t kEmptySlot = 0xffffffffu;
__device__ __forceinline__ int tile_slot_insert(uint32_t *s_key, uint32_t tile)
{
    uint32_t slot = (tile * 2654435761u) >> 20;                 // 12 bits
    for (int tries = 0; tries < 48; ++tries) {
        const uint32_t prev = atomicCAS(&s_key[slot], kEmptySlot, tile);
        if (prev == kEmptySlot || prev == tile) return (int)slot;
        slot = (slot + 1) & (kTileSlots - 1);
    }
    return -1;
}
__device__ __forceinline__ int tile_slot_find(const uint32_t *s_key, uint32_t tile)
{
    uint32_t slot = (tile * 2654435761u) >> 20;
    for (int tries = 0; tries < 48; ++tries) {
        const uint32_t k = s_key[slot];
        if (k == tile) return (int)slot;
        if (k == kEmptySlot) return -1;
        slot = (slot + 1) & (kTileSlots - 1);
    }
    return -1;
}

// K1: one thread per Gaussian (blockIdx.y = frame).  Besides the per-Gaussian state it counts, per tile, the instances the
// tile will receive (tile_count[frame][tile]): the binning that follows is a bucket sort by tile, not a global sort.
// The CTA's 256 Gaussians first count into the shared-memory tile table and then add only its occupied slots to the global counters:
// one global atomic per (CTA, touched tile) instead of one per instance, which would put a few hundred thousand atomics on a few
// hundred hot addresses that serialise in L2.
// kSH / kCov (per-frame API only, B = 1): SH colours into cc.rgb / cc.clamped, Sigma from cc.cov3D.
// kScene (composite forward): frame b holds P + sc.Ps Gaussians, the dynamic P first (per-frame means / scales, strided rotations /
// opacities, as without it), then the static set; a static Gaussian's SH colour for frame b's camera centre goes to sc.rgb[b].
// kAA: antialiased opacities (preprocess_one) for the Gaussians of the dynamic set, kAAStatic for those of the static set (kScene).
template <bool kSH = false, bool kCov = false, bool kScene = false, bool kAA = false, bool kAAStatic = false>
__global__ void __launch_bounds__(256)
preprocess_fwd_kernel(int P, int H, int W, int gx, int gy, CamSrc cam, float mod, const float *__restrict__ means3D,
                      const float *__restrict__ scales, const float *__restrict__ rots, long long rot_stride,
                      const float *__restrict__ opac, long long opac_stride, float *__restrict__ depth,
                      float2 *__restrict__ xy, float4 *__restrict__ conic_o, float *__restrict__ cov3d,
                      uint32_t *__restrict__ tiles, ushort4 *__restrict__ rect, int32_t *__restrict__ radii,
                      uint32_t *__restrict__ tile_count, ColorCov cc, SceneSet sc)
{
    const int b = blockIdx.y;
    __shared__ float view[16], proj[16];
    if (threadIdx.x < 16) view[threadIdx.x] = cam.view[(size_t)b * cam.stride + threadIdx.x];
    else if (threadIdx.x < 32) proj[threadIdx.x - 16] = cam.proj[(size_t)b * cam.stride + threadIdx.x - 16];
    __syncthreads();
    const float tanfovx = cam.tan ? cam.tan[(size_t)b * cam.stride] : cam.tanx;
    const float tanfovy = cam.tan ? cam.tan[(size_t)b * cam.stride + 1] : cam.tany;
    const int il = blockIdx.x * blockDim.x + threadIdx.x;
    ushort4 rc = make_ushort4(0, 0, 0, 0);
    if constexpr (kScene) {
        const int Pf = P + sc.Ps;
        if (il < P) {
            rc = preprocess_one<false, kAA>(il, (size_t)b * Pf + il, (size_t)b * P + il, H, W, gx, gy, view, proj, tanfovx, tanfovy, mod,
                                       means3D, scales, rots + (size_t)b * rot_stride + 4 * (size_t)il, nullptr,
                                       opac[(size_t)b * opac_stride + il], depth, xy, conic_o, cov3d, tiles, rect, radii);
        } else if (il < Pf) {
            const size_t j = (size_t)(il - P);
            rc = preprocess_one<false, kAAStatic>(il, (size_t)b * Pf + il, j, H, W, gx, gy, view, proj, tanfovx, tanfovy, mod, sc.means3D, sc.scales,
                                       sc.rotations + 4 * j, nullptr, sc.opacities[j], depth, xy, conic_o, cov3d, tiles, rect, radii);
            float r[3] = {0.f, 0.f, 0.f};
            if (rc.z > rc.x)
                sh_eval(sc.shs + j * 3 * sc.M, sc.D, sc.vec4, cam.view + (size_t)b * cam.stride + kCamPos, sc.means3D[3 * j],
                        sc.means3D[3 * j + 1], sc.means3D[3 * j + 2], r);
            float *o = sc.rgb + 3 * ((size_t)b * sc.Ps + j);
            o[0] = r[0]; o[1] = r[1]; o[2] = r[2];
        }
    } else if (il < P) {
        rc = preprocess_one<kCov, kAA>(il, (size_t)b * P + il, (size_t)b * P + il, H, W, gx, gy, view, proj, tanfovx, tanfovy, mod, means3D, scales,
                                  rots + (size_t)b * rot_stride + 4 * (size_t)il, cc.cov3D + 6 * (size_t)il,
                                  opac[(size_t)b * opac_stride + il], depth, xy, conic_o, cov3d, tiles, rect, radii);
        if constexpr (kSH)
            sh_color_fwd(cc, (size_t)il, means3D[3 * (size_t)il], means3D[3 * (size_t)il + 1], means3D[3 * (size_t)il + 2], rc.z > rc.x);
    }
    uint32_t *tc = tile_count + (size_t)b * gx * gy;
    __shared__ uint32_t s_key[kTileSlots], s_cnt[kTileSlots];
    for (int t = threadIdx.x; t < kTileSlots; t += blockDim.x) { s_key[t] = kEmptySlot; s_cnt[t] = 0u; }
    __syncthreads();
    for_each_tile_balanced(rc, gx, 0ull, [&](uint32_t tile, uint64_t) {
        const int slot = tile_slot_insert(s_key, tile);
        if (slot >= 0) atomicAdd(&s_cnt[slot], 1u);
        else atomicAdd(&tc[tile], 1u);
    });
    __syncthreads();
    for (int t = threadIdx.x; t < kTileSlots; t += blockDim.x) {
        const uint32_t c = s_cnt[t];
        if (c) atomicAdd(&tc[s_key[t]], c);
    }
}

// K2: ONE CTA scans the per-tile instance counts of all frames: tile ranges (global offsets into the instance arrays; untouched
// tiles keep (0,0) as upstream's memset leaves them), the scatter cursors, the segment index space of the backward, the
// per-frame base offsets and the overflow flag.  A tile whose range would end past the capacity gets an empty range (and the
// flag is raised): nothing downstream can overrun the buffers.  It also orders the tiles by list length (classes of
// floor(log2(count)), longest first; `order`, with status[3] = number of non-empty tiles) so that the per-tile kernels start
// their longest work first and touch empty tiles last or not at all.
__global__ void __launch_bounds__(1024)
tile_scan_kernel(int n, int T, long long capacity, const uint32_t *__restrict__ count, uint2 *__restrict__ ranges,
                 uint32_t *__restrict__ cursor, uint32_t *__restrict__ seg_start, uint32_t *__restrict__ order,
                 int32_t *__restrict__ status)
{
    using Scan = cub::BlockScan<unsigned long long, 1024>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ unsigned long long carry_c, carry_s;
    __shared__ uint32_t cls_count[33], cls_base[33];
    if (threadIdx.x == 0) { carry_c = 0; carry_s = 0; }
    if (threadIdx.x < 33) cls_count[threadIdx.x] = 0;
    __syncthreads();
    constexpr int kItems = 4;                       // tiles per thread per round: 4096 tiles per round
    for (int base = 0; base < n; base += 1024 * kItems) {
        unsigned long long c[kItems], ex[kItems], segs[kItems], sex[kItems], tot, stot;
        bool fits[kItems];
#pragma unroll
        for (int k = 0; k < kItems; ++k) { const int i = base + threadIdx.x * kItems + k; c[k] = i < n ? count[i] : 0ull; }
        Scan(tmp).ExclusiveSum(c, ex, tot);
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            const unsigned long long end = carry_c + ex[k] + c[k];
            fits[k] = end <= (unsigned long long)capacity;
            segs[k] = (fits[k] && c[k]) ? (c[k] + kSeg - 1) / kSeg : 0ull;
        }
        __syncthreads();
        Scan(tmp).ExclusiveSum(segs, sex, stot);
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            const int i = base + threadIdx.x * kItems + k;
            if (i < n) {
                const unsigned long long pos = carry_c + ex[k], end = pos + c[k];
                ranges[i] = (fits[k] && c[k]) ? make_uint2((uint32_t)pos, (uint32_t)end) : make_uint2(0u, 0u);
                cursor[i] = (uint32_t)(pos < 0xffffffffull ? pos : 0xffffffffull);
                seg_start[i] = (uint32_t)(carry_s + sex[k]);
                if (i % T == 0) status[4 + i / T] = (int32_t)(pos < 0x7fffffffull ? pos : 0x7fffffffull);
                // class 0: empty (or not fitting) tiles, class k >= 1: 2^(k-1) <= count < 2^k
                atomicAdd(&cls_count[(fits[k] && c[k]) ? 32 - __clz((uint32_t)c[k]) : 0], 1u);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) { carry_c += tot; carry_s += stot; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        status[0] = (int32_t)(carry_c < 0x7fffffffull ? carry_c : 0x7fffffffull);
        status[1] = carry_c > (unsigned long long)capacity ? 1 : 0;
        status[2] = (int32_t)carry_s;
        status[4 + n / T] = status[0];
        seg_start[n] = (uint32_t)carry_s;
        uint32_t run = 0;
        for (int k = 32; k >= 0; --k) { cls_base[k] = run; run += cls_count[k]; }    // longest class first, empties last
        status[3] = (int32_t)cls_base[0];
        static_assert(kSortSmallMax == 2048, "class boundary below assumes 2^11");
        status[13] = (int32_t)cls_base[11];           // tiles of class >= 12 (count >= 2048) come first in `order`
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += 1024) {
        const uint2 r = ranges[i];
        const uint32_t c = r.y - r.x;
        order[atomicAdd(&cls_base[c ? 32 - __clz(c) : 0], 1u)] = (uint32_t)i;
    }
}

// K3: one thread per Gaussian drops (depth bits << 32 | index) into the bucket of every tile its rect touches (large rects are
// spread over the warp, see for_each_tile_balanced).  As in K1 the CTA counts into the shared-memory tile table first, reserves ONE
// contiguous run per touched tile with a single global atomic, and hands out the places inside the run with shared-memory atomics.
__global__ void __launch_bounds__(256)
bucket_scatter_kernel(int P, int gx, int T, long long capacity, const float *__restrict__ depth,
                      const uint32_t *__restrict__ tiles, const ushort4 *__restrict__ rect, uint32_t *__restrict__ cursor,
                      uint64_t *__restrict__ bucket)
{
    const int b = blockIdx.y;
    const int il = blockIdx.x * blockDim.x + threadIdx.x;
    ushort4 rc = make_ushort4(0, 0, 0, 0);
    uint64_t key = 0;
    if (il < P) {
        const size_t i = (size_t)b * P + il;
        if (tiles[i] != 0) {
            rc = rect[i];
            key = ((uint64_t)__float_as_uint(depth[i]) << 32) | (uint32_t)il;
        }
    }
    uint32_t *cur = cursor + (size_t)b * T;
    __shared__ uint32_t s_key[kTileSlots], s_cnt[kTileSlots];   // counts, then the next place inside the CTA's run of each tile
    for (int t = threadIdx.x; t < kTileSlots; t += blockDim.x) { s_key[t] = kEmptySlot; s_cnt[t] = 0u; }
    __syncthreads();
    for_each_tile_balanced(rc, gx, 0ull, [&](uint32_t tile, uint64_t) {
        const int slot = tile_slot_insert(s_key, tile);
        if (slot >= 0) atomicAdd(&s_cnt[slot], 1u);
    });
    __syncthreads();
    for (int t = threadIdx.x; t < kTileSlots; t += blockDim.x) {
        const uint32_t c = s_cnt[t];
        if (c) s_cnt[t] = atomicAdd(&cur[s_key[t]], c);
    }
    __syncthreads();
    for_each_tile_balanced(rc, gx, key, [&](uint32_t tile, uint64_t k) {
        const int slot = tile_slot_find(s_key, tile);
        const uint32_t pos = slot >= 0 ? atomicAdd(&s_cnt[slot], 1u) : atomicAdd(&cur[tile], 1u);
        if ((long long)pos < capacity) bucket[pos] = k;
    });
}

// Squared distance from a Gaussian's centre beyond which it is certain that the compositing loop skips it
// (alpha = min(0.99, o exp(power)) < 1/255):  power <= -0.5 lmin |d|^2 with lmin the smaller eigenvalue of the conic.
// Conservative by construction (1 % slack on alpha, lmin pushed down by its round-off, 0.1 % on the radius), so culling a
// (Gaussian, sub-tile) pair never changes a result: every pair that could pass the exact per-pixel tests is still
// evaluated with the exact arithmetic.  Returns -1 (always culled) for opacity below the threshold, +inf (never culled) for
// an indefinite or NaN conic.
__device__ __forceinline__ float cull_radius2(const float4 co)
{
    if (co.w <= 0.f) return -1.f;
    const float thr = logf(255.f * co.w) + 0.01f;
    if (thr <= 0.f) return -1.f;
    const float mid = 0.5f * (co.x + co.z), hd = 0.5f * (co.x - co.z);
    const float lmin = mid - sqrtf(hd * hd + co.y * co.y) - 1e-5f * fabsf(mid);
    if (!(lmin > 0.f)) return INFINITY;
    return 2.002f * thr / lmin;
}

// Squared distance from point c to the pixel rectangle [x0,x1] x [y0,y1] (0 inside).
__device__ __forceinline__ float rect_dist2(const float2 c, float x0, float x1, float y0, float y1)
{
    const float ex = fmaxf(fmaxf(x0 - c.x, c.x - x1), 0.f), ey = fmaxf(fmaxf(y0 - c.y, c.y - y1), 0.f);
    return ex * ex + ey * ey;
}

// Bitonic sort of n2 (power of two) 64-bit keys in shared memory by the whole CTA.
__device__ __forceinline__ void bitonic_sort_smem(uint64_t *keys, int n2)
{
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < (n2 >> 1); t += blockDim.x) {
                // t-th compare-exchange of this step: partner indices i < l differ in bit j
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                const int l = i | j;
                const uint64_t a = keys[i], c = keys[l];
                const bool up = (i & k) == 0;
                if ((a > c) == up) { keys[i] = c; keys[l] = a; }
            }
            __syncthreads();
        }
}

// K4: one CTA per (frame, tile) sorts the tile's bucket by (depth bits, Gaussian index) — upstream's order — and emits, in list
// order, the Gaussian index and the packed record the compositing kernels stream.  Buckets longer than kSortMax are sorted
// kSortMax keys at a time (written back in place) and merged by rank: keys are unique, so an element's final position is
// the number of smaller keys, i.e. the sum of its lower bounds in the sorted runs.
// kScene (composite forward, P = Pd + Ps per frame): colours of indices below Pd come from colors [B,Pd,3], the others from K1's
// per-frame scene rgb [B,Ps,3].
// kZ (for K6's depth variant, the only reader of recC.w): recC.w is the entry's view depth z, the key's high word (K1's depth,
// exact); otherwise 0.  A template parameter because holding the high word changes the short instance's register allocation.
template <int kThreads, int kMax, bool kLong, bool kScene = false, bool kZ = false>
__global__ void __launch_bounds__(kThreads)
tile_sort_kernel(int P, int T, int BT, const int32_t *__restrict__ status, const uint32_t *__restrict__ order,
                 const uint2 *__restrict__ ranges, const uint32_t *__restrict__ seg_start,
                 uint64_t *__restrict__ bucket, const float2 *__restrict__ xy, const float4 *__restrict__ conic_o,
                 const float *__restrict__ colors, uint32_t *__restrict__ point_list, float4 *__restrict__ recA,
                 float4 *__restrict__ recB, float4 *__restrict__ recC, uint32_t *__restrict__ seg_tile,
                 uint32_t *__restrict__ tile_maxc, const float *__restrict__ scene_rgb, int Pd)
{
    extern __shared__ uint64_t s_keys[];
    using BinScan = cub::BlockScan<uint32_t, kThreads>;
    constexpr int kBins = 2 * kThreads;              // at most two depth bins per thread
    __shared__ typename BinScan::TempStorage s_scan;
    __shared__ uint32_t s_hist[kBins + 1], s_off[kBins + 1], s_red[3];
    if (kLong)
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < BT; i += gridDim.x * blockDim.x) tile_maxc[i] = 0u;
    // `order` lists the tiles by decreasing length class: the first status[13] have >= kSortSmallMax entries (this kernel's kLong
    // instance), the rest up to status[3] are shorter (the 128-thread instance)
    const int first = kLong ? 0 : status[13], last = kLong ? status[13] : status[3];
    for (int it = first + blockIdx.x; it < last; it += gridDim.x) {
        const int blk = (int)order[it];
        const uint2 r = ranges[blk];
        const int n = (int)(r.y - r.x);
        const size_t gbase = (size_t)(blk / T) * P;      // this frame's Gaussians
        const uint32_t s0 = seg_start[blk];
        for (int i = threadIdx.x; i < (n + kSeg - 1) / kSeg; i += blockDim.x) seg_tile[s0 + i] = (uint32_t)blk;
        // kScene: colour row of this frame's Gaussian idx
        auto scene_col = [&](uint32_t idx) {
            const size_t f = (size_t)(blk / T);
            return idx < (uint32_t)Pd ? colors + 3 * (f * Pd + idx) : scene_rgb + 3 * (f * (P - Pd) + (idx - Pd));
        };

        auto rec_z = [](uint64_t key) { return kZ ? __uint_as_float((uint32_t)(key >> 32)) : 0.f; };
        auto emit = [&](int rank, uint64_t key) {
            const uint32_t idx = (uint32_t)key;
            const size_t g = gbase + idx, o = (size_t)r.x + rank;
            const float2 c = xy[g];
            const float4 co = conic_o[g];
            point_list[o] = idx;
            recA[o] = make_float4(c.x, c.y, cull_radius2(co), __uint_as_float(idx));
            recB[o] = co;
            if constexpr (kScene) {
                const float *cp = scene_col(idx);
                recC[o] = make_float4(cp[0], cp[1], cp[2], rec_z(key));
            } else {
                recC[o] = make_float4(colors[3 * g], colors[3 * g + 1], colors[3 * g + 2], rec_z(key));
            }
        };

        if (n <= kMax) {
            // Bucket-then-insertion: one counting pass over linear depth bins (about 8 entries each) puts every key within a few
            // places of its final position, one thread per bin finishes it by insertion — a fraction of the shared-memory traffic of
            // a full bitonic network.  Bins are monotone in depth, ties inside a bin are ordered by the full (depth bits, index) key,
            // so the result is the same total order.  Degenerate depth distributions (a bin above kMaxBin entries, e.g. many
            // equal depths) fall back to the bitonic network on the same buffer.
            // The thread's keys (at most kPer = kMax / kThreads) are read from global memory ONCE, all loads in flight together, and
            // stay in registers through the min/max, histogram and scatter passes: the kernel is bound by memory latency, not
            // bandwidth (ncu: long_scoreboard on top, 12-14 % issue-active), so what counts is the number of dependent round trips.
            constexpr int kMaxBin = 48;
            constexpr int kPer = kMax / kThreads;
            uint64_t key[kPer];
#pragma unroll
            for (int k = 0; k < kPer; ++k) { const int i = threadIdx.x + k * kThreads; key[k] = i < n ? bucket[r.x + i] : ~0ull; }
            const int nb = n >= 64 ? min(kBins, max(32, n >> 3)) : 0;
            bool binned = false, filled = false;
            if (nb) {
                uint32_t lo = 0xffffffffu, hi = 0u;
#pragma unroll
                for (int k = 0; k < kPer; ++k)
                    if (threadIdx.x + k * kThreads < n) { const uint32_t d = (uint32_t)(key[k] >> 32); lo = min(lo, d); hi = max(hi, d); }
                for (int i = threadIdx.x; i < kBins + 1; i += blockDim.x) s_hist[i] = 0;
                if (threadIdx.x == 0) { s_red[0] = 0xffffffffu; s_red[1] = 0u; s_red[2] = 0u; }
                __syncthreads();
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
                if ((threadIdx.x & 31) == 0) { atomicMin(&s_red[0], lo); atomicMax(&s_red[1], hi); }
                __syncthreads();
                const float dmin = __uint_as_float(s_red[0]), dmax = __uint_as_float(s_red[1]);      // depths are positive: bit order = value order
                if (dmax > dmin) {
                    const float scale = (float)nb / (dmax - dmin);
                    auto bin_of = [&](uint64_t kk) { return min(nb - 1, (int)((__uint_as_float((uint32_t)(kk >> 32)) - dmin) * scale)); };
#pragma unroll
                    for (int k = 0; k < kPer; ++k)
                        if (threadIdx.x + k * kThreads < n) atomicAdd(&s_hist[bin_of(key[k])], 1u);
                    __syncthreads();
                    // exclusive scan of the bin counts (nb <= 2 per thread) and their maximum
                    uint32_t c0 = 2 * threadIdx.x < nb ? s_hist[2 * threadIdx.x] : 0u, c1 = 2 * threadIdx.x + 1 < nb ? s_hist[2 * threadIdx.x + 1] : 0u;
                    uint32_t ex;
                    BinScan(s_scan).ExclusiveSum(c0 + c1, ex);
                    if (max(c0, c1) > kMaxBin) s_red[2] = 1u;
                    __syncthreads();
                    if (2 * threadIdx.x < nb) { s_off[2 * threadIdx.x] = ex; s_hist[2 * threadIdx.x] = ex; }
                    if (2 * threadIdx.x + 1 < nb) { s_off[2 * threadIdx.x + 1] = ex + c0; s_hist[2 * threadIdx.x + 1] = ex + c0; }
                    if (threadIdx.x == 0) s_off[nb] = (uint32_t)n;
                    __syncthreads();
#pragma unroll
                    for (int k = 0; k < kPer; ++k)
                        if (threadIdx.x + k * kThreads < n) s_keys[atomicAdd(&s_hist[bin_of(key[k])], 1u)] = key[k];
                    filled = true;
                    __syncthreads();
                    if (s_red[2] == 0u) {
                        for (int bi = threadIdx.x; bi < nb; bi += blockDim.x) {
                            const int b0 = (int)s_off[bi], b1 = (int)s_off[bi + 1];
                            for (int i = b0 + 1; i < b1; ++i) {
                                const uint64_t kk = s_keys[i];
                                int j = i - 1;
                                while (j >= b0 && s_keys[j] > kk) { s_keys[j + 1] = s_keys[j]; --j; }
                                s_keys[j + 1] = kk;
                            }
                        }
                        __syncthreads();
                        binned = true;
                    }
                }
            }
            if (!binned) {
                int n2 = 32;
                while (n2 < n) n2 <<= 1;
                if (!filled) {
#pragma unroll
                    for (int k = 0; k < kPer; ++k) { const int i = threadIdx.x + k * kThreads; if (i < n) s_keys[i] = key[k]; }
                }
                for (int i = n + threadIdx.x; i < n2; i += blockDim.x) s_keys[i] = ~0ull;
                __syncthreads();
                bitonic_sort_smem(s_keys, n2);
            }
            // emit four list entries per thread at a time: the 4 x 5 gathers they need are independent and in flight together
            for (int i0 = 0; i0 < n; i0 += 4 * kThreads) {
                uint64_t kk[4]; float2 c[4]; float4 co[4]; float col[4][3];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = i0 + threadIdx.x + u * kThreads;
                    kk[u] = i < n ? s_keys[i] : 0ull;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const size_t g = gbase + (uint32_t)kk[u];
                    c[u] = xy[g]; co[u] = conic_o[g];
                    if constexpr (kScene) {
                        const float *cp = scene_col((uint32_t)kk[u]);
                        col[u][0] = cp[0]; col[u][1] = cp[1]; col[u][2] = cp[2];
                    } else {
                        col[u][0] = colors[3 * g]; col[u][1] = colors[3 * g + 1]; col[u][2] = colors[3 * g + 2];
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = i0 + threadIdx.x + u * kThreads;
                    if (i < n) {
                        const size_t o = (size_t)r.x + i;
                        point_list[o] = (uint32_t)kk[u];
                        recA[o] = make_float4(c[u].x, c[u].y, cull_radius2(co[u]), __uint_as_float((uint32_t)kk[u]));
                        recB[o] = co[u];
                        // kZ: the depth word is re-read from shared memory rather than held through the gathers (no spill)
                        recC[o] = make_float4(col[u][0], col[u][1], col[u][2], rec_z(kZ ? s_keys[i] : 0ull));
                    }
                }
            }
            __syncthreads();                 // s_keys is reloaded by the next tile
            continue;
        }
        for (int c0 = 0; c0 < n; c0 += kMax) {
            const int m = min(kMax, n - c0);
            int n2 = 32;
            while (n2 < m) n2 <<= 1;
            for (int i = threadIdx.x; i < n2; i += blockDim.x) s_keys[i] = i < m ? bucket[r.x + c0 + i] : ~0ull;
            __syncthreads();
            bitonic_sort_smem(s_keys, n2);
            for (int i = threadIdx.x; i < m; i += blockDim.x) bucket[r.x + c0 + i] = s_keys[i];
            __syncthreads();
        }
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const uint64_t key = bucket[r.x + i];
            int rank = 0;
            for (int c0 = 0; c0 < n; c0 += kMax) {
                const uint64_t *run = bucket + r.x + c0;
                int lo = 0, hi = min(kMax, n - c0);
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (run[mid] < key) lo = mid + 1; else hi = mid;
                }
                rank += lo;
            }
            emit(rank, key);
        }
        __syncthreads();
    }
}

// exp(x) for the compositing kernels, x in [-5.6, 0] (anything smaller ends below the 1/255 alpha cut-off): one FMUL + MUFU.EX2 instead
// of the ~10-instruction library expf.  Relative error <= ~6e-7 (0.5 ulp of x*log2(e) plus ex2.approx's 2 ulp), three orders of
// magnitude inside the 1e-4 image bar; forward and backward use the same function, so the replay stays consistent.
__device__ __forceinline__ float comp_exp(float x)
{
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x * 1.4426950408889634f));
    return r;
}

// One compositing step of pixel (pxf, pyf) against a staged record: SURVEY.md §8 a-8 K6 (power > 0 skip, alpha = min(0.99, o e^p),
// alpha < 1/255 skip, test_T < 1e-4 -> done and not blended), written without branches so that two consecutive entries
// overlap in the pipeline (only T carries a dependence from one to the next).
struct PixState {
    float T, C0, C1, C2;
    uint32_t last;
    bool done;
};

__device__ __forceinline__ float entry_alpha(const float4 a, const float4 co, float pxf, float pyf, bool &ok)
{
    const float dx = a.x - pxf, dy = a.y - pyf;
    const float power = -0.5f * (co.x * dx * dx + co.z * dy * dy) - co.y * dx * dy;
    const float alpha = fminf(0.99f, co.w * comp_exp(power));
    ok = !(power > 0.f) && !(alpha < 1.0f / 255.0f);
    return alpha;
}

__device__ __forceinline__ float blend(PixState &p, float alpha, bool ok, const float4 rgb, uint32_t pos1)
{
    const float test_T = p.T * (1.f - alpha);
    const bool live = ok && !p.done;
    const bool stop = live && test_T < 0.0001f;
    const bool take = live && !stop;
    const float w = take ? alpha * p.T : 0.f;
    p.C0 += rgb.x * w; p.C1 += rgb.y * w; p.C2 += rgb.z * w;
    p.T = take ? test_T : p.T;
    p.last = take ? pos1 : p.last;
    p.done = p.done || stop;
    return w;
}

// The sets of ga_rasterb_forward_mattes: entry idx of a frame belongs to set k when first[k] <= idx < first[k+1]; sets k >= K
// are empty (first[k] = first[K]), and so is every index at or above first[K] (the rest of the dynamic set, the scene's).
constexpr int kMaxSets = 8;
struct MatteSets {
    uint32_t first[kMaxSets + 1];
    int K;
    float *out;              // [B, K, H, W]
};

// Adds an entry's blending weight to the accumulator of its set: unrolled selects keep the accumulators in registers.  The add
// is never contracted with the product that formed w, so matte k equals the colour channel an indicator colour of set k gives.
__device__ __forceinline__ void matte_add(float (&mt)[kMaxSets], const MatteSets &ms, uint32_t idx, float w)
{
#pragma unroll
    for (int k = 0; k < kMaxSets; ++k) mt[k] = __fadd_rn(mt[k], (idx >= ms.first[k] && idx < ms.first[k + 1]) ? w : 0.f);
}

// K6: one CTA per (frame, 16x16 tile), one warp per 8x4-pixel sub-tile, one lane per pixel.  The warps of a CTA do not
// synchronise with each other: each walks the tile's record stream 32 entries at a time (next chunk prefetched into
// registers), tests the 32 against its sub-tile in parallel (one per lane, cull_radius2 precomputed by the sort kernel),
// stages them in its own slice of shared memory and composites the ballot's survivors in list order, two at a time.
// At every 256th list position it stores each pixel's (T, C) — the state the backward's segment CTAs start from.
// kMattes: also sums, per pixel and per set of `ms`, the weights alpha T its set's entries add, and writes them to ms.out; every
// other output is the same.
// kDepth: also writes depth [B,2,H,W] over the blended entries (z = recC.w): plane 0 the mean D / (1 - T), D = sum of w z
// accumulated as the colour channels are (so D is the red channel a colour (z, 0, 0) gives), 0 where nothing was blended;
// plane 1 the median, the z of the entry whose blend takes T from above 0.5 to at most 0.5, 0 where the final T > 0.5.  An
// entry that is not blended leaves T unchanged, so the T crossing alone selects a blended one; the 1e-4 stop cannot pre-empt
// the crossing, since alpha <= 0.99 puts T below 0.01 before it can fire.
// With kDepth and a depth state (d_ckpt, d_final non-NULL: the training forward), it also stores each pixel's running D next to
// the (T, C) checkpoints and D at the end, the state the depth backward's segments start from.
template <bool kMattes, bool kDepth>
__global__ void __launch_bounds__(kBlock)
render_fwd_kernel(int H, int W, int gx, int T_tiles, const uint32_t *__restrict__ order, const uint2 *__restrict__ ranges,
                  const uint32_t *__restrict__ seg_start,
                  const float4 *__restrict__ recA, const float4 *__restrict__ recB, const float4 *__restrict__ recC,
                  const float *__restrict__ bg, float4 *__restrict__ ckpt, float *__restrict__ final_T,
                  uint32_t *__restrict__ n_contrib, float4 *__restrict__ final_state, uint32_t *__restrict__ tile_maxc,
                  float *__restrict__ out, const MatteSets ms, float *__restrict__ depth, float *__restrict__ d_ckpt,
                  float *__restrict__ d_final)
{
    __shared__ float4 s_a[kBlock / 32][32], s_b[kBlock / 32][32], s_c[kBlock / 32][32];

    const int blk = (int)order[blockIdx.x];           // longest tile lists first
    const int b = blk / T_tiles, tile = blk - b * T_tiles;
    const int tx = tile % gx, ty = tile / gx;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sx = tx * kTile + (warp & 1) * 8, sy = ty * kTile + (warp >> 1) * 4;
    const int px = sx + (lane & 7), py = sy + (lane >> 3);
    const float x0f = (float)sx, x1f = (float)(sx + 7), y0f = (float)sy, y1f = (float)(sy + 3);
    const bool inside = px < W && py < H;
    const float pxf = (float)px, pyf = (float)py;
    const uint2 range = ranges[blk];
    const int n = (int)(range.y - range.x);
    const int nchunks = (n + 31) >> 5;
    float4 *ck = ckpt + (size_t)seg_start[blk] * kBlock + tid;

    PixState p{1.f, 0.f, 0.f, 0.f, 0u, !inside};
    float mt[kMaxSets];
    if constexpr (kMattes) {
#pragma unroll
        for (int k = 0; k < kMaxSets; ++k) mt[k] = 0.f;
    }
    float dsum = 0.f, dmed = 0.f;
    float4 fa = make_float4(0.f, 0.f, -1.f, 0.f), fb = fa, fc = fa;
    if (lane < n) { fa = recA[range.x + lane]; fb = recB[range.x + lane]; fc = recC[range.x + lane]; }

    bool all_done = __all_sync(0xffffffffu, p.done);          // a sub-tile entirely outside the image
    for (int c = 0; c < nchunks && !all_done; ++c) {
        if ((c & 7) == 0) {
            ck[(size_t)(c >> 3) * kBlock] = make_float4(p.T, p.C0, p.C1, p.C2);
            if constexpr (kDepth)
                if (d_ckpt) d_ckpt[((size_t)seg_start[blk] + (c >> 3)) * kBlock + tid] = dsum;
        }
        const float4 a = fa, bq = fb, cq = fc;
        const int kn = (c + 1) * 32 + lane;          // prefetch the next chunk behind this one's compositing
        if (kn < n) { fa = recA[range.x + kn]; fb = recB[range.x + kn]; fc = recC[range.x + kn]; }
        const bool hit = (c * 32 + lane < n) && !(rect_dist2(make_float2(a.x, a.y), x0f, x1f, y0f, y1f) > a.z);
        uint32_t mask = __ballot_sync(0xffffffffu, hit);
        if (mask) {
            __syncwarp();
            s_a[warp][lane] = a; s_b[warp][lane] = bq; s_c[warp][lane] = cq;
            __syncwarp();
            const uint32_t base1 = (uint32_t)(c * 32) + 1u;
            while (mask) {
                const int j0 = __ffs(mask) - 1;
                mask &= mask - 1;
                const bool two = mask != 0;
                const int j1 = two ? __ffs(mask) - 1 : j0;
                mask &= mask - 1;                                   // no-op on 0
                bool ok0, ok1;
                const float al0 = entry_alpha(s_a[warp][j0], s_b[warp][j0], pxf, pyf, ok0);
                const float al1 = entry_alpha(s_a[warp][j1], s_b[warp][j1], pxf, pyf, ok1);
                const float T0 = p.T;
                const float w0 = blend(p, al0, ok0, s_c[warp][j0], base1 + j0);
                const float T1 = p.T;
                const float w1 = blend(p, al1, ok1 && two, s_c[warp][j1], base1 + j1);
                if constexpr (kDepth) {
                    const float z0 = s_c[warp][j0].w, z1 = s_c[warp][j1].w;
                    dsum += z0 * w0;
                    dsum += z1 * w1;
                    dmed = (T0 > 0.5f && T1 <= 0.5f) ? z0 : dmed;
                    dmed = (T1 > 0.5f && p.T <= 0.5f) ? z1 : dmed;
                }
                if constexpr (kMattes) {
                    matte_add(mt, ms, __float_as_uint(s_a[warp][j0].w), w0);
                    matte_add(mt, ms, __float_as_uint(s_a[warp][j1].w), w1);
                }
            }
            all_done = __all_sync(0xffffffffu, p.done);
        }
    }
    const size_t HW = (size_t)H * W;
    if (inside) {
        const size_t pid = (size_t)b * HW + (size_t)py * W + px;
        final_T[pid] = p.T;
        n_contrib[pid] = p.last;
        float *o = out + (size_t)b * 3 * HW + (size_t)py * W + px;
        o[0] = p.C0 + p.T * bg[0];
        o[HW] = p.C1 + p.T * bg[1];
        o[2 * HW] = p.C2 + p.T * bg[2];
        if constexpr (kMattes) {
            float *mo = ms.out + (size_t)b * ms.K * HW + (size_t)py * W + px;
#pragma unroll
            for (int k = 0; k < kMaxSets; ++k)
                if (k < ms.K) mo[(size_t)k * HW] = mt[k];
        }
        if constexpr (kDepth) {
            float *dp = depth + (size_t)b * 2 * HW + (size_t)py * W + px;
            dp[0] = p.last ? __fdiv_rn(dsum, __fsub_rn(1.f, p.T)) : 0.f;
            dp[HW] = dmed;
        }
    }
    final_state[(size_t)blk * kBlock + tid] = make_float4(p.T, p.C0, p.C1, p.C2);
    if constexpr (kDepth)
        if (d_final) d_final[(size_t)blk * kBlock + tid] = dsum;
    uint32_t m = p.last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0 && m) atomicMax(&tile_maxc[blk], m);
}

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Reduce 8 per-lane values across the warp with 9 shuffles (recursive halving: after the xor-16 / 8 / 4 steps a lane
// holds ONE of the eight sums over 8 lanes, the xor-2 / 1 steps finish it).  Returns the sum of value
// `idx = 4*bit4(lane) + 2*bit3(lane) + bit2(lane)` over all 32 lanes (replicated over the lane's 4-lane group).
__device__ __forceinline__ float warp_reduce8(float (&v)[8], int lane)
{
    const bool h4 = lane & 16, h3 = lane & 8, h2 = lane & 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float send = h4 ? v[i] : v[i + 4];
        const float recv = __shfl_xor_sync(0xffffffffu, send, 16);
        v[i] = (h4 ? v[i + 4] : v[i]) + recv;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float send = h3 ? v[i] : v[i + 2];
        const float recv = __shfl_xor_sync(0xffffffffu, send, 8);
        v[i] = (h3 ? v[i + 2] : v[i]) + recv;
    }
    {
        const float send = h2 ? v[0] : v[1];
        const float recv = __shfl_xor_sync(0xffffffffu, send, 4);
        v[0] = (h2 ? v[1] : v[0]) + recv;
    }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 2);
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
    return v[0];
}

// K7: one CTA per 256-entry SEGMENT of a tile list; all segments of all tiles of all frames run in parallel.  Inside a
// segment the replay is upstream's: back to front, T <- T / (1 - alpha), the colour behind the entry by the recurrence
// acc <- last_alpha * last_colour + (1 - last_alpha) * acc.  A pixel whose blended entries continue past the segment starts
// from the forward's checkpoint behind it: T = T_ckpt and acc = (C_final - C_ckpt) / T_ckpt (the colour composited behind the
// checkpoint, un-premultiplied); a pixel whose last contributor lies inside the segment starts from (T_final, 0) as upstream
// does.  Per-Gaussian gradients are reduced warp-wide with shuffles (9 for the 8 components GaussianAvatar consumes), across
// the CTA's eight warps in shared memory, then leave as one vector reduction per (segment entry, array).
// kDepth: also the gradient of the mean depth m = D / A (plane 0 of depth, A = 1 - T_final) given g = dL_dm per pixel.  The depth
// is a fourth colour channel of the same recurrence: colour z = recC.w, upstream gradient g / A, and the pixel's own m as its
// "background" (the normalisation's dA/dalpha term has bg_dot's shape), so dL/dalpha gains (g / A) [T (z - zacc) - m T_final /
// (1 - alpha)] and each entry's dL/dz = (g / A) alpha T goes to d_z [B,P].  A restarted segment starts from the forward's stored D:
// zacc = (D_final - D_ckpt) / T_ckpt.
template <bool kOpacity, bool kDepth = false>
__global__ void __launch_bounds__(kBlock)
render_bwd_kernel(int H, int W, int gx, int T_tiles, int P, const int32_t *__restrict__ status,
                  const uint32_t *__restrict__ seg_tile, const uint32_t *__restrict__ seg_start,
                  const uint2 *__restrict__ ranges, const uint32_t *__restrict__ tile_maxc,
                  const float4 *__restrict__ recA, const float4 *__restrict__ recB, const float4 *__restrict__ recC,
                  const float4 *__restrict__ ckpt, const float *__restrict__ bg, const float4 *__restrict__ final_state,
                  const uint32_t *__restrict__ n_contrib, const float *__restrict__ dL_dout,
                  float2 *__restrict__ d_mean2D, float4 *__restrict__ d_conic_op, float *__restrict__ d_colors,
                  const float *__restrict__ dL_dm, const float *__restrict__ depth, const float *__restrict__ d_ckpt,
                  const float *__restrict__ d_final, float *__restrict__ d_z)
{
    __shared__ float4 s_a[kSeg], s_b[kSeg], s_c[kSeg];
    __shared__ float s_acc[kDepth ? 10 : 9][kSeg + 1];      // + 1: the 8 lanes that own a Gaussian's 8 sums hit 8 different banks

    const int g = blockIdx.x;
    if (g >= status[2]) return;
    const int blk = (int)seg_tile[g];
    const int seg = g - (int)seg_start[blk];
    const uint32_t maxc = tile_maxc[blk];
    const uint32_t lo = (uint32_t)seg * kSeg;                 // first list position of this segment
    if (lo >= maxc) return;                                   // nothing blended at or behind this segment: uniform for the CTA
    const uint2 range = ranges[blk];
    const uint32_t hi = min(min(range.y - range.x, lo + kSeg), maxc);   // positions [lo, hi) are replayed, back to front
    const int cnt = (int)(hi - lo);

    const int b = blk / T_tiles, tile = blk - b * T_tiles;
    const int tx = tile % gx, ty = tile / gx;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sx = tx * kTile + (warp & 1) * 8, sy = ty * kTile + (warp >> 1) * 4;
    const int px = sx + (lane & 7), py = sy + (lane >> 3);
    const float x0f = (float)sx, x1f = (float)(sx + 7), y0f = (float)sy, y1f = (float)(sy + 3);
    const bool inside = px < W && py < H;
    const float pxf = (float)px, pyf = (float)py;
    const size_t HW = (size_t)H * W, pid = (size_t)py * W + px;

    // stage the segment back to front: slot j holds list position hi - 1 - j
    if (tid < cnt) {
        const size_t o = (size_t)range.x + (hi - 1 - tid);
        s_a[tid] = recA[o]; s_b[tid] = recB[o]; s_c[tid] = recC[o];
    }
#pragma unroll
    for (int k = 0; k < (kDepth ? 10 : 9); ++k) s_acc[k][tid] = 0.f;

    const float4 fs = final_state[(size_t)blk * kBlock + tid];
    const float T_final = inside ? fs.x : 0.f;
    const uint32_t last_contributor = inside ? n_contrib[(size_t)b * HW + pid] : 0u;
    float dpix0 = 0.f, dpix1 = 0.f, dpix2 = 0.f;
    if (inside) {
        const float *d = dL_dout + (size_t)b * 3 * HW + pid;
        dpix0 = d[0]; dpix1 = d[HW]; dpix2 = d[2 * HW];
    }
    float bg_dot = bg[0] * dpix0 + bg[1] * dpix1 + bg[2] * dpix2;
    float gA = 0.f;                                // kDepth: dL/dm / A, 0 where nothing was blended (m = 0, A = 0)
    if constexpr (kDepth) {
        if (last_contributor) {
            const float m = depth[(size_t)b * 2 * HW + pid];
            gA = dL_dm[(size_t)b * HW + pid] / __fsub_rn(1.f, T_final);
            bg_dot += m * gA;
        }
    }
    float T = T_final, acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, accz = 0.f;
    if (last_contributor > lo + kSeg) {            // blended entries continue behind this segment
        const size_t ci = ((size_t)seg_start[blk] + seg + 1) * kBlock + tid;
        const float4 ck = ckpt[ci];
        const float inv = 1.f / ck.x;
        T = ck.x;
        acc0 = (fs.y - ck.y) * inv; acc1 = (fs.z - ck.z) * inv; acc2 = (fs.w - ck.w) * inv;
        if constexpr (kDepth) accz = (d_final[(size_t)blk * kBlock + tid] - d_ckpt[ci]) * inv;
    }
    float lc0 = 0.f, lc1 = 0.f, lc2 = 0.f, lcz = 0.f, last_alpha = 0.f;
    const float ddelx_dx = 0.5f * (float)W, ddely_dy = 0.5f * (float)H;
    const int vidx = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);   // component this lane ends up owning
    __syncthreads();

    for (int j0 = 0; j0 < cnt; j0 += 32) {
        const int jt = j0 + lane;
        bool hit = false;
        if (jt < cnt) { const float4 a = s_a[jt]; hit = !(rect_dist2(make_float2(a.x, a.y), x0f, x1f, y0f, y1f) > a.z); }
        uint32_t mask = __ballot_sync(0xffffffffu, hit);
        while (mask) {
            const int j = j0 + __ffs(mask) - 1;
            mask &= mask - 1;
            const uint32_t index = hi - 1 - (uint32_t)j;            // 0-based position in the tile list
            bool active = index < last_contributor;
            float4 co; float dx = 0.f, dy = 0.f, G = 0.f, alpha = 0.f;
            if (active) {
                const float4 a = s_a[j]; co = s_b[j];
                dx = a.x - pxf; dy = a.y - pyf;
                const float power = -0.5f * (co.x * dx * dx + co.z * dy * dy) - co.y * dx * dy;
                if (power > 0.f) active = false;
                else {
                    G = comp_exp(power);
                    alpha = fminf(0.99f, co.w * G);
                    if (alpha < 1.0f / 255.0f) active = false;
                }
            }
            if (!__any_sync(0xffffffffu, active)) continue;
            float v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = 0.f;
            float vo = 0.f, vz = 0.f;
            if (active) {
                T = T / (1.f - alpha);
                const float dchannel_dcolor = alpha * T;
                const float4 col = s_c[j];
                acc0 = last_alpha * lc0 + (1.f - last_alpha) * acc0; lc0 = col.x;
                acc1 = last_alpha * lc1 + (1.f - last_alpha) * acc1; lc1 = col.y;
                acc2 = last_alpha * lc2 + (1.f - last_alpha) * acc2; lc2 = col.z;
                float dL_dalpha = (col.x - acc0) * dpix0 + (col.y - acc1) * dpix1 + (col.z - acc2) * dpix2;
                if constexpr (kDepth) {
                    accz = last_alpha * lcz + (1.f - last_alpha) * accz; lcz = col.w;
                    dL_dalpha += (col.w - accz) * gA;
                    vz = dchannel_dcolor * gA;
                }
                v[0] = dchannel_dcolor * dpix0; v[1] = dchannel_dcolor * dpix1; v[2] = dchannel_dcolor * dpix2;
                dL_dalpha *= T;
                last_alpha = alpha;
                dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
                const float dL_dG = co.w * dL_dalpha;
                const float gdx = G * dx, gdy = G * dy;
                const float dG_ddelx = -gdx * co.x - gdy * co.y;
                const float dG_ddely = -gdy * co.z - gdx * co.y;
                v[3] = dL_dG * dG_ddelx * ddelx_dx;
                v[4] = dL_dG * dG_ddely * ddely_dy;
                v[5] = -0.5f * gdx * dx * dL_dG;
                v[6] = -0.5f * gdx * dy * dL_dG;
                v[7] = -0.5f * gdy * dy * dL_dG;
                vo = G * dL_dalpha;
            }
            const float red = warp_reduce8(v, lane);
            if ((lane & 3) == 0) atomicAdd(&s_acc[vidx][j], red);
            if (kOpacity) {
                vo = warp_sum(vo);
                if (lane == 0) atomicAdd(&s_acc[8][j], vo);
            }
            if constexpr (kDepth) {
                vz = warp_sum(vz);
                if (lane == 0) atomicAdd(&s_acc[9][j], vz);
            }
        }
    }
    __syncthreads();
    if (tid < cnt) {
        const size_t gi = (size_t)b * P + __float_as_uint(s_a[tid].w);
        float a[kDepth ? 10 : 9];
#pragma unroll
        for (int k = 0; k < (kDepth ? 10 : 9); ++k) a[k] = s_acc[k][tid];
        if (a[0] != 0.f) atomicAdd(&d_colors[3 * gi], a[0]);
        if (a[1] != 0.f) atomicAdd(&d_colors[3 * gi + 1], a[1]);
        if (a[2] != 0.f) atomicAdd(&d_colors[3 * gi + 2], a[2]);
        // 8- and 16-byte vector reductions (sm_90+): one L2 atomic per float2 / float4 instead of one per component
        if (a[3] != 0.f || a[4] != 0.f)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(&d_mean2D[gi]), "f"(a[3]), "f"(a[4]) : "memory");
        if (a[5] != 0.f || a[6] != 0.f || a[7] != 0.f || (kOpacity && a[8] != 0.f))
            red_add_v4(&d_conic_op[gi].x, a[5], a[6], a[7], kOpacity ? a[8] : 0.f);
        if constexpr (kDepth)
            if (a[9] != 0.f) atomicAdd(&d_z[gi], a[9]);
    }
}

// Fused K8 (conic -> cov2D -> cov3D / mean) + K9 (mean2D -> mean3D, cov3D -> scale / rotation): one thread per Gaussian.
// kSH: also the SH colour backward (d_sh, direction term of d_means3D); kCov: dL/dSigma goes to cc.d_cov3D and the scale /
// rotation chain is skipped (per-frame API only, B = 1).  kZ: d_means3D also gets dL/dz [B,P] (the depth backward's d_z) times
// the view matrix's z row, the derivative of the view-space z K1 computes.
// kAA: the backward of K1's antialiased opacity o rho (preprocess_one).  rho is recomputed here from this kernel's own 2D
// covariance, o is the stored opacity conic_o.w over it (rho >= 0.005), dL/do = gO rho and, where the clamp is inactive,
// dL/drho = gO o goes through rho = sqrt(r), r = det0 / det1 into the 2D-covariance gradients.
template <bool kSH = false, bool kCov = false, bool kZ = false, bool kAA = false>
__global__ void __launch_bounds__(256)
preprocess_bwd_kernel(int P, int H, int W, CamSrc cam, float mod, const float *__restrict__ means3D,
                      const float *__restrict__ scales, const float *__restrict__ rots, long long rot_stride,
                      const int32_t *__restrict__ radii, const float *__restrict__ cov3d,
                      const float2 *__restrict__ d_mean2D, const float4 *__restrict__ d_conic_op,
                      float *__restrict__ d_means3D, float *__restrict__ d_scales, float *__restrict__ d_rots,
                      float *__restrict__ d_opac, float *__restrict__ d_means2D_out, ColorCov cc, const float *__restrict__ d_z,
                      const float4 *__restrict__ conic_o)
{
    const int fb = blockIdx.y;
    __shared__ float view[16], proj[16];
    if (threadIdx.x < 16) view[threadIdx.x] = cam.view[(size_t)fb * cam.stride + threadIdx.x];
    else if (threadIdx.x < 32) proj[threadIdx.x - 16] = cam.proj[(size_t)fb * cam.stride + threadIdx.x - 16];
    __syncthreads();
    const float tanfovx = cam.tan ? cam.tan[(size_t)fb * cam.stride] : cam.tanx;
    const float tanfovy = cam.tan ? cam.tan[(size_t)fb * cam.stride + 1] : cam.tany;
    const int il = blockIdx.x * blockDim.x + threadIdx.x;
    if (il >= P) return;
    const size_t i = (size_t)fb * P + il;
    const float *rq = rots + (size_t)fb * rot_stride + 4 * (size_t)il;
    const size_t i3 = 3 * (size_t)i;
    const float4 gco = d_conic_op[i];
    const float2 g2 = d_mean2D[i];
    if (d_opac && (!kAA || radii[i] <= 0)) d_opac[i] = gco.w;     // kAA: gO rho, written below for a visible Gaussian
    if (d_means2D_out) { d_means2D_out[i3] = g2.x; d_means2D_out[i3 + 1] = g2.y; d_means2D_out[i3 + 2] = 0.f; }
    if (radii[i] <= 0) {
        d_means3D[i3] = d_means3D[i3 + 1] = d_means3D[i3 + 2] = 0.f;
        if constexpr (kSH) sh_row_store(cc.d_sh + i * 3 * cc.M, 3 * cc.M, cc.vec4, [](int) { return 0.f; });
        if constexpr (kCov) {
#pragma unroll
            for (int k = 0; k < 6; ++k) cc.d_cov3D[6 * i + k] = 0.f;
        } else {
            d_scales[i3] = d_scales[i3 + 1] = d_scales[i3 + 2] = 0.f;
            if (d_rots) { d_rots[4 * (size_t)i] = d_rots[4 * (size_t)i + 1] = d_rots[4 * (size_t)i + 2] = d_rots[4 * (size_t)i + 3] = 0.f; }
        }
        return;
    }
    const float px = means3D[i3], py = means3D[i3 + 1], pz = means3D[i3 + 2];
    const float tvx = xf_row(view, 0, px, py, pz), tvy = xf_row(view, 1, px, py, pz), tvz = xf_row(view, 2, px, py, pz);
    const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
    const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
    const float txtz = tvx / tvz, tytz = tvy / tvz;
    const float tx = fminf(limx, fmaxf(-limx, txtz)) * tvz, ty = fminf(limy, fmaxf(-limy, tytz)) * tvz;
    const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    const float tz = 1.f / tvz, tz2 = tz * tz, tz3 = tz2 * tz;
    const float J00 = fx * tz, J02 = -fx * tx * tz2, J11 = fy * tz, J12 = -fy * ty * tz2;
    float m0[3], m1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        m0[k] = view[k * 4 + 0] * J00 + view[k * 4 + 2] * J02;
        m1[k] = view[k * 4 + 1] * J11 + view[k * 4 + 2] * J12;
    }
    const float *c3 = cov3d + 6 * (size_t)i;
    const float Sg[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
    float v0[3], v1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        v0[k] = Sg[k][0] * m0[0] + Sg[k][1] * m0[1] + Sg[k][2] * m0[2];
        v1[k] = Sg[k][0] * m1[0] + Sg[k][1] * m1[1] + Sg[k][2] * m1[2];
    }
    const float a = m0[0] * v0[0] + m0[1] * v0[1] + m0[2] * v0[2] + 0.3f;
    const float b = m0[0] * v1[0] + m0[1] * v1[1] + m0[2] * v1[2];
    const float c = m1[0] * v1[0] + m1[1] * v1[1] + m1[2] * v1[2] + 0.3f;
    const float gA = gco.x, gBh = gco.y, gC = gco.z;  // gBh: half-convention off-diagonal (see a-9 spec)
    const float denom = a * c - b * b;
    const float denom2inv = 1.f / (denom * denom + 0.0000001f);
    float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
    if (denom2inv != 0.f) {
        dL_da = denom2inv * (-c * c * gA + 2.f * b * c * gBh + (denom - a * c) * gC);
        dL_dc = denom2inv * (-a * a * gC + 2.f * a * b * gBh + (denom - a * c) * gA);
        dL_db = denom2inv * 2.f * (b * c * gA - (denom + 2.f * b * b) * gBh + a * b * gC);
    }
    if constexpr (kAA) {
        // r = det0 / det1.  The numerators of dr/d(a0, c0, b) det1^2 are expanded so that no two large terms cancel:
        // c0 det1 - det0 c = 0.3 (c0^2 + b^2) + 0.09 c0, a0 det1 - det0 a = 0.3 (a0^2 + b^2) + 0.09 a0, det1 - det0 = 0.3 (a0 + c0) + 0.09.
        const float a0 = m0[0] * v0[0] + m0[1] * v0[1] + m0[2] * v0[2];      // a and c before the dilation
        const float c0 = m1[0] * v1[0] + m1[1] * v1[1] + m1[2] * v1[2];
        const float det0 = a0 * c0 - b * b;
        const float r = det0 / denom;
        const float rho = sqrtf(fmaxf(2.5e-5f, r));
        if (d_opac) d_opac[i] = gco.w * rho;
        if (r > 2.5e-5f) {
            const float o = conic_o[i].w / rho;
            const float g = gco.w * o * 0.5f / (rho * denom * denom);     // dL/drho drho/dr / det1^2
            dL_da += g * (0.3f * (c0 * c0 + b * b) + 0.09f * c0);
            dL_dc += g * (0.3f * (a0 * a0 + b * b) + 0.09f * a0);
            dL_db -= g * 2.f * b * (0.3f * (a0 + c0) + 0.09f);
        }
    }
    float dc[6];
    dc[0] = m0[0] * m0[0] * dL_da + m0[0] * m1[0] * dL_db + m1[0] * m1[0] * dL_dc;
    dc[3] = m0[1] * m0[1] * dL_da + m0[1] * m1[1] * dL_db + m1[1] * m1[1] * dL_dc;
    dc[5] = m0[2] * m0[2] * dL_da + m0[2] * m1[2] * dL_db + m1[2] * m1[2] * dL_dc;
    dc[1] = 2.f * m0[0] * m0[1] * dL_da + (m0[0] * m1[1] + m0[1] * m1[0]) * dL_db + 2.f * m1[0] * m1[1] * dL_dc;
    dc[2] = 2.f * m0[0] * m0[2] * dL_da + (m0[0] * m1[2] + m0[2] * m1[0]) * dL_db + 2.f * m1[0] * m1[2] * dL_dc;
    dc[4] = 2.f * m0[2] * m0[1] * dL_da + (m0[1] * m1[2] + m0[2] * m1[1]) * dL_db + 2.f * m1[1] * m1[2] * dL_dc;
    float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float dm0 = 2.f * v0[k] * dL_da + v1[k] * dL_db;
        const float dm1 = 2.f * v1[k] * dL_dc + v0[k] * dL_db;
        dJ00 += view[k * 4 + 0] * dm0; dJ02 += view[k * 4 + 2] * dm0;
        dJ11 += view[k * 4 + 1] * dm1; dJ12 += view[k * 4 + 2] * dm1;
    }
    const float dL_dtx = x_grad_mul * -fx * tz2 * dJ02;
    const float dL_dty = y_grad_mul * -fy * tz2 * dJ12;
    const float dL_dtz = -fx * tz2 * dJ00 - fy * tz2 * dJ11 + (2.f * fx * tx) * tz3 * dJ02 + (2.f * fy * ty) * tz3 * dJ12;
    float dmean[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) dmean[k] = view[k * 4 + 0] * dL_dtx + view[k * 4 + 1] * dL_dty + view[k * 4 + 2] * dL_dtz;

    const float hx = xf_row(proj, 0, px, py, pz), hy = xf_row(proj, 1, px, py, pz), hw = xf_row(proj, 3, px, py, pz);
    const float m_w = 1.f / (hw + 0.0000001f);
    const float mul1 = hx * m_w * m_w, mul2 = hy * m_w * m_w;
#pragma unroll
    for (int k = 0; k < 3; ++k)
        dmean[k] += (proj[4 * k + 0] * m_w - proj[4 * k + 3] * mul1) * g2.x + (proj[4 * k + 1] * m_w - proj[4 * k + 3] * mul2) * g2.y;
    if constexpr (kZ) {
        const float dz = d_z[i];
#pragma unroll
        for (int k = 0; k < 3; ++k) dmean[k] += view[k * 4 + 2] * dz;
    }
    if constexpr (kSH) sh_color_bwd(cc, i, px, py, pz, dmean);
    d_means3D[i3] = dmean[0]; d_means3D[i3 + 1] = dmean[1]; d_means3D[i3 + 2] = dmean[2];
    if constexpr (kCov) {
#pragma unroll
        for (int k = 0; k < 6; ++k) cc.d_cov3D[6 * i + k] = dc[k];
        return;
    }

    const float sv[3] = {mod * scales[i3], mod * scales[i3 + 1], mod * scales[i3 + 2]};
    const float qr = rq[0], qx = rq[1], qy = rq[2], qz = rq[3];
    float Rm[3][3];
    quat_to_rot(qr, qx, qy, qz, Rm);
    const float dS[3][3] = {{dc[0], 0.5f * dc[1], 0.5f * dc[2]}, {0.5f * dc[1], dc[3], 0.5f * dc[4]}, {0.5f * dc[2], 0.5f * dc[4], dc[5]}};
    float dM[3][3];
#pragma unroll
    for (int a2 = 0; a2 < 3; ++a2)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float t = 0.f;
#pragma unroll
            for (int j = 0; j < 3; ++j) t += (sv[a2] * Rm[j][a2]) * dS[j][k];
            dM[a2][k] = 2.f * t;
        }
#pragma unroll
    for (int a2 = 0; a2 < 3; ++a2) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) t += Rm[k][a2] * dM[a2][k];
        d_scales[i3 + a2] = mod * t;
    }
    if (d_rots) {
        float dR[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int a2 = 0; a2 < 3; ++a2) dR[k][a2] = sv[a2] * dM[a2][k];
        d_rots[4 * (size_t)i] = 2.f * (-qz * dR[0][1] + qy * dR[0][2] + qz * dR[1][0] - qx * dR[1][2] - qy * dR[2][0] + qx * dR[2][1]);
        d_rots[4 * (size_t)i + 1] = 2.f * (qy * dR[0][1] + qz * dR[0][2] + qy * dR[1][0] - 2.f * qx * dR[1][1] - qr * dR[1][2] + qz * dR[2][0] + qr * dR[2][1] - 2.f * qx * dR[2][2]);
        d_rots[4 * (size_t)i + 2] = 2.f * (-2.f * qy * dR[0][0] + qx * dR[0][1] + qr * dR[0][2] + qx * dR[1][0] + qz * dR[1][2] - qr * dR[2][0] + qz * dR[2][1] - 2.f * qy * dR[2][2]);
        d_rots[4 * (size_t)i + 3] = 2.f * (-2.f * qz * dR[0][0] - qr * dR[0][1] + qx * dR[0][2] + qr * dR[1][0] - 2.f * qz * dR[1][1] + qy * dR[1][2] + qx * dR[2][0] + qy * dR[2][1]);
    }
}

int check_dims(int B, int P, int H, int W)
{
    GA_REQUIRE(B >= 1 && B <= 8, "bad frame count B=%d (1..8)", B);
    GA_REQUIRE(P >= 0 && H > 0 && W > 0, "bad raster dims P=%d H=%d W=%d", P, H, W);
    GA_REQUIRE(cdiv(W, kTile) <= 65535 && cdiv(H, kTile) <= 65535, "image too large");
    GA_REQUIRE((long long)B * cdiv(W, kTile) * cdiv(H, kTile) < (1ll << 30), "too many tiles");
    return GA_OK;
}
int check_settings(const GaRasterSettings *s)
{
    GA_REQUIRE(s != nullptr, "settings is NULL");
    return check_dims(1, s->P, s->H, s->W);
}

struct FwdArgs {
    const float *means3D, *colors, *scales, *rotations, *opacities, *bg;
    long long rot_stride, opac_stride;
    float mod;
    bool aa, aa_static;      // antialiased opacities for the dynamic / static (scene) set
};

// f(std::true_type{}) or f(std::false_type{}): nested, it picks a kernel's template instance from run-time flags.
template <class F>
auto with_bool(bool b, F f)
{
    return b ? f(std::true_type{}) : f(std::false_type{});
}

// The batched API's cameras: kCamStride floats per frame, tan(fov / 2) read from the array.
CamSrc batch_cams(const float *cams) { return CamSrc{cams, cams + 16, cams + 32, kCamStride, 0.f, 0.f}; }

// K1 + K2 for all frames.  cc selects the K1 variant (all zero: precomputed colours, Sigma from scales / rotations); a scene
// selects the composite K1, with d.P = P + Ps Gaussians per frame.
int launch_preprocess(const Dims &d, const CamSrc &cam, const FwdArgs &a, const ColorCov &cc, long long capacity, const GeomViews &g,
                      const ImgViews &iv, int32_t *radii, cudaStream_t stream, const SceneSet *scene = nullptr)
{
    const size_t BT = (size_t)d.B * d.T;
    GA_CHECK_CUDA(cudaMemsetAsync(iv.count, 0, sizeof(uint32_t) * BT, stream));
    if (d.P > 0) {
        ProfScope _ps("preprocess_fwd_kernel", stream);
        auto *k1 = with_bool(a.aa, [&](auto aa) {
            return scene ? with_bool(a.aa_static, [&](auto aas) { return preprocess_fwd_kernel<false, false, true, aa, aas>; })
                         : with_bool(cc.shs != nullptr, [&](auto sh) {
                               return with_bool(cc.cov3D != nullptr, [&](auto cov) { return preprocess_fwd_kernel<sh, cov, false, aa>; });
                           });
        });
        k1<<<dim3(cdiv(d.P, 256), d.B), 256, 0, stream>>>(scene ? d.P - scene->Ps : d.P, d.H, d.W, d.gx, d.gy, cam, a.mod, a.means3D,
                 a.scales, a.rotations, a.rot_stride, a.opacities, a.opac_stride, g.depth, g.xy, g.conic_o, g.cov3d, g.tiles, g.rect, radii,
                 iv.count, cc, scene ? *scene : SceneSet{});
        GA_CHECK_LAUNCH("preprocess_fwd_kernel");
    }
    {
        ProfScope _ps("tile_scan_kernel", stream);
        tile_scan_kernel<<<1, 1024, 0, stream>>>((int)BT, d.T, capacity, iv.count, iv.ranges, iv.cursor, iv.seg_start, iv.order, iv.status);
    }
    GA_CHECK_LAUNCH("tile_scan_kernel");
    return GA_OK;
}

// The tile sort's long-segment (kLong) or short-segment instance for a forward with or without a scene and a depth pass.
template <bool kLong>
auto tile_sort_for(bool scene, bool depth)
{
    constexpr int threads = kLong ? kSortThreads : kSortSmallThreads, max = kLong ? kSortMax : kSortSmallMax;
    return with_bool(scene, [&](auto sc) { return with_bool(depth, [&](auto z) { return tile_sort_kernel<threads, max, kLong, sc, z>; }); });
}

// K3 + K4 + K6 for all frames (a scene: the composite K4, d.P = P + Ps; mattes and / or depth: K6's variant that writes them).
int launch_binning_and_render(const Dims &d, const FwdArgs &a, long long capacity, const GeomViews &g, const ImgViews &iv, const BinViews &bv,
                              float *out_color, cudaStream_t stream, const SceneSet *scene = nullptr, const MatteSets *mattes = nullptr,
                              float *depth = nullptr, const DepthState *dstate = nullptr)
{
    static PerDeviceOnce attr_set;
    if (attr_set.first())
        for (int k = 0; k < 4; ++k)      // k = (depth, scene)
            GA_CHECK_CUDA(cudaFuncSetAttribute(tile_sort_for<true>(k & 1, k & 2), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kSortMax * (int)sizeof(uint64_t)));
    const float *scene_rgb = scene ? scene->rgb : nullptr;
    const int Pd = scene ? d.P - scene->Ps : d.P;
    auto *sort_long = tile_sort_for<true>(scene != nullptr, depth != nullptr);
    auto *sort_short = tile_sort_for<false>(scene != nullptr, depth != nullptr);
    const int BT = d.B * d.T;
    if (d.P > 0) {
        {
            ProfScope _ps("bucket_scatter_kernel", stream);
            bucket_scatter_kernel<<<dim3(cdiv(d.P, 256), d.B), 256, 0, stream>>>(d.P, d.gx, d.T, capacity, g.depth, g.tiles, g.rect, iv.cursor,
                                                                                bv.bucket);
        }
        GA_CHECK_LAUNCH("bucket_scatter_kernel");
    }
    {
        ProfScope _ps("tile_sort_kernel", stream);
        sort_long<<<min(BT, 3 * num_sms()), kSortThreads, kSortMax * sizeof(uint64_t), stream>>>(
                 d.P, d.T, BT, iv.status, iv.order, iv.ranges, iv.seg_start, bv.bucket, g.xy, g.conic_o, a.colors, bv.point_list, bv.recA, bv.recB,
                 bv.recC, bv.seg_tile, iv.tile_maxc, scene_rgb, Pd);
        count_launch();
        sort_short<<<min(BT, 12 * num_sms()), kSortSmallThreads, kSortSmallMax * sizeof(uint64_t), stream>>>(
                 d.P, d.T, BT, iv.status, iv.order, iv.ranges, iv.seg_start, bv.bucket, g.xy, g.conic_o, a.colors, bv.point_list, bv.recA, bv.recB,
                 bv.recC, bv.seg_tile, iv.tile_maxc, scene_rgb, Pd);
    }
    GA_CHECK_LAUNCH("tile_sort_kernel");
    {
        static const char *const names[2][2] = {{"render_fwd_kernel", "render_fwd_depth_kernel"}, {"render_fwd_mattes_kernel", "render_fwd_mattes_depth_kernel"}};
        ProfScope _ps(names[mattes != nullptr][depth != nullptr], stream);
        auto *k6 = with_bool(mattes != nullptr, [&](auto m) { return with_bool(depth != nullptr, [&](auto z) { return render_fwd_kernel<m, z>; }); });
        k6<<<BT, kBlock, 0, stream>>>(d.H, d.W, d.gx, d.T, iv.order, iv.ranges, iv.seg_start, bv.recA, bv.recB, bv.recC, a.bg, bv.ckpt,
                                      iv.final_T, iv.n_contrib, iv.final_state, iv.tile_maxc, out_color, mattes ? *mattes : MatteSets{},
                                      depth, dstate ? dstate->ckpt : nullptr, dstate ? dstate->final : nullptr);
    }
    GA_CHECK_LAUNCH("render_fwd_kernel");
    return GA_OK;
}

struct BwdArgs {
    const float *means3D, *colors, *scales, *rotations, *bg, *dL_dout;
    long long rot_stride;
    float mod;
    float *d_means3D, *d_colors, *d_scales, *d_rotations, *d_opacities, *d_means2D;
    bool aa;                 // the forward stored antialiased opacities
};

size_t bwd_scratch_bytes(size_t BP)
{
    const size_t n = BP > 0 ? BP : 1;
    return align_up(n * sizeof(float2)) + align_up(n * sizeof(float4));
}

// The depth backward's scratch: bwd_scratch_bytes' d_mean2D and d_conic_op, then d_z [B*P].
size_t depth_bwd_scratch_bytes(size_t BP) { return bwd_scratch_bytes(BP) + align_up((BP > 0 ? BP : 1) * sizeof(float)); }

// The inputs of the depth backward: dL/dm [B,H,W], the forward's depth [B,2,H,W] and its depth state, with the sizes the caller
// gave for that state and for the backward's scratch.
struct DepthBwd {
    const float *dL_dm, *depth;
    DepthState state;
    size_t state_bytes, scratch_bytes;
};

// K7 + fused K8/K9.  cc selects the K8/K9 variant as in launch_preprocess; with SH, K7's d_colors is dL/drgb (cc.d_rgb).  dz (batched
// API, no SH / cov3D): the depth variants, with d_z behind d_conic_op in the scratch (depth_bwd_scratch_bytes).
int launch_backward(const Dims &d, const CamSrc &cam, const BwdArgs &a, ColorCov cc, const int32_t *radii, const GeomViews &g,
                    const ImgViews &iv, const BinViews &bv, void *scratch, cudaStream_t stream, const DepthBwd *dz = nullptr)
{
    const size_t BP = (size_t)d.B * d.P;
    Carver sc(scratch);
    float2 *d_mean2D = sc.take<float2>(BP);
    float4 *d_conic_op = sc.take<float4>(BP);
    float *d_z = dz ? sc.take<float>(BP) : nullptr;
    GA_CHECK_CUDA(cudaMemsetAsync(scratch, 0, dz ? depth_bwd_scratch_bytes(BP) : bwd_scratch_bytes(BP), stream));
    GA_CHECK_CUDA(cudaMemsetAsync(a.d_colors, 0, sizeof(float) * 3 * BP, stream));
    {
        ProfScope _ps(dz ? "render_bwd_depth_kernel" : "render_bwd_kernel", stream);
        auto *k7 = with_bool(a.d_opacities != nullptr, [&](auto op) { return with_bool(dz != nullptr, [&](auto z) { return render_bwd_kernel<op, z>; }); });
        k7<<<(int)bv.max_segments, kBlock, 0, stream>>>(d.H, d.W, d.gx, d.T, d.P, iv.status, bv.seg_tile, iv.seg_start, iv.ranges, iv.tile_maxc,
                                                        bv.recA, bv.recB, bv.recC, bv.ckpt, a.bg, iv.final_state, iv.n_contrib, a.dL_dout,
                                                        d_mean2D, d_conic_op, a.d_colors, dz ? dz->dL_dm : nullptr, dz ? dz->depth : nullptr,
                                                        dz ? dz->state.ckpt : nullptr, dz ? dz->state.final : nullptr, d_z);
    }
    GA_CHECK_LAUNCH("render_bwd_kernel");
    {
        ProfScope _ps("preprocess_bwd_kernel", stream);
        cc.d_rgb = a.d_colors;
        auto *k89 = with_bool(a.aa, [&](auto aa) {
            return dz ? preprocess_bwd_kernel<false, false, true, aa>
                      : with_bool(cc.shs != nullptr, [&](auto sh) {
                            return with_bool(cc.cov3D != nullptr, [&](auto cov) { return preprocess_bwd_kernel<sh, cov, false, aa>; });
                        });
        });
        k89<<<dim3(cdiv(d.P, 256), d.B), 256, 0, stream>>>(d.P, d.H, d.W, cam, a.mod, a.means3D, a.scales, a.rotations, a.rot_stride,
                 radii, g.cov3d, d_mean2D, d_conic_op, a.d_means3D, a.d_scales, a.d_rotations, a.d_opacities, a.d_means2D, cc, d_z,
                 g.conic_o);
    }
    GA_CHECK_LAUNCH("preprocess_bwd_kernel");
    return GA_OK;
}

constexpr long long kNoCapacity = 0x7fffffffll;   // per-frame API: the host sizes the binning buffer after reading the count

}  // namespace
}  // namespace ga

using namespace ga;

// ---- per-frame API (upstream's call shape: the host reads the instance count to size the binning buffer) -------------------
extern "C" size_t ga_raster_geom_bytes(int32_t P) { return carve_geom(nullptr, (size_t)(P > 0 ? P : 0)).total; }
extern "C" size_t ga_raster_img_bytes(int32_t H, int32_t W) { return carve_img(nullptr, make_dims(1, 0, H, W)).total; }
extern "C" size_t ga_raster_binning_bytes(int64_t R, int32_t H, int32_t W) { return carve_bin(nullptr, R, make_dims(1, 0, H, W)).total; }
extern "C" size_t ga_raster_bwd_scratch_bytes(int32_t P) { return bwd_scratch_bytes((size_t)(P > 0 ? P : 0)); }

// Validates a GaRasterColorCov (NULL: neither mode) and turns it into the kernels' ColorCov.
static int color_cov_of(const GaRasterColorCov *in, ColorCov &out)
{
    out = ColorCov{};
    if (!in) return GA_OK;
    if (in->shs) {
        GA_REQUIRE(in->sh_degree >= 0 && in->sh_degree <= 3, "sh_degree %d outside 0..3", (int)in->sh_degree);
        GA_REQUIRE(in->sh_coeffs >= (in->sh_degree + 1) * (in->sh_degree + 1), "sh_coeffs %d < (sh_degree + 1)^2 = %d", (int)in->sh_coeffs,
                   (int)((in->sh_degree + 1) * (in->sh_degree + 1)));
        GA_REQUIRE(in->campos && in->rgb && in->clamped, "shs given without campos / rgb / clamped");
        out.shs = in->shs;
        out.D = in->sh_degree;
        out.M = in->sh_coeffs;
        out.vec4 = in->sh_coeffs % 4 == 0 && reinterpret_cast<uintptr_t>(in->shs) % 16 == 0;
        out.campos = in->campos;
        out.rgb = in->rgb;
        out.clamped = in->clamped;
    }
    out.cov3D = in->cov3D_precomp;
    return GA_OK;
}

extern "C" int ga_raster_forward_preprocess_ex(const GaRasterSettings *s, const GaRasterColorCov *cc_in, const float *means3D,
                                               const float *scales, const float *rotations, const float *opacities,
                                               const float *viewmatrix, const float *projmatrix, void *geom, void *img, int32_t *radii,
                                               int64_t *num_rendered_host, void *stream_)
{
    if (int rc = check_settings(s)) return rc;
    GA_REQUIRE(num_rendered_host && img, "NULL pointer argument");
    *num_rendered_host = 0;
    ColorCov cc;
    if (int rc = color_cov_of(cc_in, cc)) return rc;
    GA_REQUIRE(s->P == 0 || (means3D && (cc.cov3D || (scales && rotations)) && opacities && viewmatrix && projmatrix && geom && radii),
               "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const Dims d = make_dims(1, s->P, s->H, s->W);
    GeomViews g = carve_geom(geom, (size_t)s->P);
    ImgViews iv = carve_img(img, d);
    const CamSrc cam{viewmatrix, projmatrix, nullptr, 0, s->tanfovx, s->tanfovy};
    const FwdArgs a{means3D, nullptr, scales, rotations, opacities, nullptr, 0, 0, s->scale_modifier, s->antialiasing != 0};
    if (int rc = launch_preprocess(d, cam, a, cc, kNoCapacity, g, iv, radii, stream)) return rc;
    int32_t total = 0;
    GA_CHECK_CUDA(cudaMemcpyAsync(&total, iv.status, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    GA_CHECK_CUDA(cudaStreamSynchronize(stream));
    *num_rendered_host = (int64_t)total;
    return GA_OK;
}

extern "C" int ga_raster_forward_preprocess(const GaRasterSettings *s, const float *means3D, const float *scales,
                                            const float *rotations, const float *opacities, const float *viewmatrix,
                                            const float *projmatrix, void *geom, void *img, int32_t *radii,
                                            int64_t *num_rendered_host, void *stream_)
{
    return ga_raster_forward_preprocess_ex(s, nullptr, means3D, scales, rotations, opacities, viewmatrix, projmatrix, geom, img, radii,
                                           num_rendered_host, stream_);
}

extern "C" int ga_raster_forward_render(const GaRasterSettings *s, const float *colors, const float *bg, void *geom, void *binning,
                                        size_t binning_bytes, int64_t R, void *img, float *out_color, void *stream_)
{
    if (int rc = check_settings(s)) return rc;
    GA_REQUIRE(bg && img && out_color && binning, "NULL pointer argument");
    GA_REQUIRE(R >= 0 && R < (int64_t)kNoCapacity, "num_rendered out of range: %lld", (long long)R);
    GA_REQUIRE(s->P == 0 || (colors && geom), "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const Dims d = make_dims(1, s->P, s->H, s->W);
    BinViews bv = carve_bin(binning, R, d);
    if (bv.total > binning_bytes) {
        set_error("binning buffer too small: need %zu bytes, have %zu", bv.total, binning_bytes);
        return GA_ERR_CAPACITY;
    }
    const FwdArgs a{nullptr, colors, nullptr, nullptr, nullptr, bg, 0, 0, s->scale_modifier};
    return launch_binning_and_render(d, a, R, carve_geom(geom, (size_t)s->P), carve_img(img, d), bv, out_color, stream);
}

extern "C" int ga_raster_backward_ex(const GaRasterSettings *s, const GaRasterColorCov *cc_in, const float *means3D,
                                     const float *colors, const float *scales, const float *rotations, const float *bg,
                                     const float *viewmatrix, const float *projmatrix, const int32_t *radii, const void *geom,
                                     const void *binning, const void *img, int64_t R, const float *dL_dout, void *scratch,
                                     float *d_means3D, float *d_colors, float *d_scales, float *d_rotations, float *d_opacities,
                                     float *d_means2D, float *d_sh, float *d_cov3D, void *stream_)
{
    if (int rc = check_settings(s)) return rc;
    ColorCov cc;
    if (int rc = color_cov_of(cc_in, cc)) return rc;
    if (s->P == 0) return GA_OK;
    GA_REQUIRE(means3D && (colors || cc.shs) && (cc.cov3D || (scales && rotations && d_scales)) && bg && viewmatrix && projmatrix &&
                   radii && geom && img && binning && dL_dout && scratch && d_means3D && d_colors,
               "NULL pointer argument");
    GA_REQUIRE(!cc.shs || d_sh, "shs given without d_sh");
    GA_REQUIRE(!cc.cov3D || d_cov3D, "cov3D_precomp given without d_cov3D");
    cc.vec4 = cc.vec4 && reinterpret_cast<uintptr_t>(d_sh) % 16 == 0;
    cc.d_sh = d_sh;
    cc.d_cov3D = d_cov3D;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const Dims d = make_dims(1, s->P, s->H, s->W);
    const CamSrc cam{viewmatrix, projmatrix, nullptr, 0, s->tanfovx, s->tanfovy};
    const BwdArgs a{means3D, colors, scales, rotations, bg, dL_dout, 0, s->scale_modifier, d_means3D, d_colors, d_scales, d_rotations,
                    d_opacities, d_means2D, s->antialiasing != 0};
    return launch_backward(d, cam, a, cc, radii, carve_geom(const_cast<void *>(geom), (size_t)s->P),
                           carve_img(const_cast<void *>(img), d), carve_bin(const_cast<void *>(binning), R, d), scratch, stream);
}

extern "C" int ga_raster_backward(const GaRasterSettings *s, const float *means3D, const float *colors, const float *scales,
                                  const float *rotations, const float *bg, const float *viewmatrix, const float *projmatrix,
                                  const int32_t *radii, const void *geom, const void *binning, const void *img, int64_t R,
                                  const float *dL_dout, void *scratch, float *d_means3D, float *d_colors, float *d_scales,
                                  float *d_rotations, float *d_opacities, float *d_means2D, void *stream_)
{
    return ga_raster_backward_ex(s, nullptr, means3D, colors, scales, rotations, bg, viewmatrix, projmatrix, radii, geom, binning, img, R,
                                 dL_dout, scratch, d_means3D, d_colors, d_scales, d_rotations, d_opacities, d_means2D, nullptr, nullptr,
                                 stream_);
}

// ---- batched API: every frame of a step in one set of launches, no host read-back ------------------------------------------
static int check_batch(const GaRasterBatchDesc *d)
{
    GA_REQUIRE(d != nullptr, "batch descriptor is NULL");
    if (int rc = check_dims(d->B, d->P, d->H, d->W)) return rc;
    GA_REQUIRE(d->capacity >= 0 && d->capacity < (int64_t)kNoCapacity, "capacity out of range: %lld", (long long)d->capacity);
    GA_REQUIRE((d->rot_stride == 0 || d->rot_stride == 4ll * d->P) && (d->opac_stride == 0 || d->opac_stride == (long long)d->P),
               "rot_stride / opac_stride must be 0 (shared) or one frame");
    return GA_OK;
}
extern "C" size_t ga_rasterb_geom_bytes(int32_t B, int32_t P) { return carve_geom(nullptr, (size_t)B * (size_t)(P > 0 ? P : 0)).total; }
extern "C" size_t ga_rasterb_img_bytes(int32_t B, int32_t H, int32_t W) { return carve_img(nullptr, make_dims(B, 0, H, W)).total; }
extern "C" size_t ga_rasterb_binning_bytes(int32_t B, int32_t H, int32_t W, int64_t capacity)
{
    return carve_bin(nullptr, capacity, make_dims(B, 0, H, W)).total;
}
extern "C" size_t ga_rasterb_bwd_scratch_bytes(int32_t B, int32_t P) { return bwd_scratch_bytes((size_t)B * (size_t)(P > 0 ? P : 0)); }
extern "C" const int32_t *ga_rasterb_status(int32_t B, int32_t H, int32_t W, const void *img)
{
    return carve_img(const_cast<void *>(img), make_dims(B, 0, H, W)).status;
}

namespace ga {
namespace {
__global__ void stamp_serial_kernel(int32_t *status, const int32_t *serial)
{
    status[kStatusInts - 1] = *serial;
}
}  // namespace
}  // namespace ga

// Copies the 16 status words (the caller's serial number stamped into word 15) to pinned host memory behind the forward, on
// `stream`.  Plain cudaMemcpyAsync: capturable in a CUDA graph, no event involved — the host recognises a fresh copy by its serial.
extern "C" int ga_rasterb_status_to_host(int32_t B, int32_t H, int32_t W, void *img, const int32_t *serial_dev, int32_t *host16,
                                         void *stream_)
{
    if (int rc = check_dims(B, 0, H, W)) return rc;
    GA_REQUIRE(img && serial_dev && host16, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int32_t *status = carve_img(img, make_dims(B, 0, H, W)).status;
    stamp_serial_kernel<<<1, 1, 0, stream>>>(status, serial_dev);
    GA_CHECK_LAUNCH("stamp_serial_kernel");
    GA_CHECK_CUDA(cudaMemcpyAsync(host16, status, sizeof(int32_t) * kStatusInts, cudaMemcpyDeviceToHost, stream));
    return GA_OK;
}

// The batched forward (bd checked by the caller): scene NULL renders the dynamic set alone, a scene (even with Ps = 0) through the
// composite kernels; mattes NULL writes no mattes, depth NULL no depth.  Every check runs before the first launch.
static int forward_batch(const GaRasterBatchDesc *bd, const GaRasterScene *scene, const MatteSets *mattes, float *depth,
                         const float *cams, const float *bg, const float *means3D, const float *colors, const float *scales,
                         const float *rotations, const float *opacities, void *geom, void *img, void *binning, int32_t *radii,
                         float *out_color, cudaStream_t stream, const DepthState *dstate = nullptr)
{
    int Pt = bd->P;
    if (scene) {
        GA_REQUIRE(scene->Ps >= 0 && (long long)bd->P + scene->Ps <= 0x7fffffffll, "bad static count Ps=%d (P=%d)", (int)scene->Ps, (int)bd->P);
        Pt += scene->Ps;
        if (int rc = check_dims(bd->B, Pt, bd->H, bd->W)) return rc;
    }
    GA_REQUIRE(cams && bg && img && binning && out_color, "NULL pointer argument");
    GA_REQUIRE(bd->P == 0 || (means3D && colors && scales && rotations && opacities), "NULL pointer argument");
    GA_REQUIRE(Pt == 0 || (geom && radii), "NULL pointer argument");
    SceneSet sc{};
    if (scene && scene->Ps > 0) {
        GA_REQUIRE(scene->means3D && scene->scales && scene->rotations && scene->opacities && scene->shs && scene->rgb,
                   "NULL pointer in the scene descriptor");
        GA_REQUIRE(scene->sh_degree >= 0 && scene->sh_degree <= 3, "scene sh_degree %d outside 0..3", (int)scene->sh_degree);
        GA_REQUIRE(scene->sh_coeffs >= (scene->sh_degree + 1) * (scene->sh_degree + 1), "scene sh_coeffs %d < (sh_degree + 1)^2 = %d",
                   (int)scene->sh_coeffs, (int)((scene->sh_degree + 1) * (scene->sh_degree + 1)));
        sc = SceneSet{scene->means3D, scene->scales, scene->rotations, scene->opacities, scene->shs, scene->Ps, scene->sh_degree,
                      scene->sh_coeffs, scene->sh_coeffs % 4 == 0 && reinterpret_cast<uintptr_t>(scene->shs) % 16 == 0, scene->rgb};
    }
    const SceneSet *set = scene ? &sc : nullptr;
    const Dims d = make_dims(bd->B, Pt, bd->H, bd->W);
    GeomViews g = carve_geom(geom, (size_t)d.B * d.P);
    ImgViews iv = carve_img(img, d);
    BinViews bv = carve_bin(binning, bd->capacity, d);
    const FwdArgs a{means3D, colors, scales, rotations, opacities, bg, bd->rot_stride, bd->opac_stride, bd->scale_modifier,
                    bd->antialiasing != 0, scene && scene->antialiasing != 0};
    if (int rc = launch_preprocess(d, batch_cams(cams), a, ColorCov{}, bd->capacity, g, iv, radii, stream, set)) return rc;
    return launch_binning_and_render(d, a, bd->capacity, g, iv, bv, out_color, stream, set, mattes, depth, dstate);
}

extern "C" int ga_rasterb_forward(const GaRasterBatchDesc *bd, const float *cams, const float *bg, const float *means3D,
                                  const float *colors, const float *scales, const float *rotations, const float *opacities,
                                  void *geom, void *img, void *binning, int32_t *radii, float *out_color, void *stream_)
{
    if (int rc = check_batch(bd)) return rc;
    return forward_batch(bd, nullptr, nullptr, nullptr, cams, bg, means3D, colors, scales, rotations, opacities, geom, img, binning, radii, out_color,
                         static_cast<cudaStream_t>(stream_));
}

extern "C" int ga_rasterb_forward_scene(const GaRasterBatchDesc *bd, const GaRasterScene *scene, const float *cams, const float *bg,
                                        const float *means3D, const float *colors, const float *scales, const float *rotations,
                                        const float *opacities, void *geom, void *img, void *binning, int32_t *radii, float *out_color,
                                        void *stream_)
{
    if (int rc = check_batch(bd)) return rc;
    GA_REQUIRE(scene != nullptr, "scene descriptor is NULL");
    return forward_batch(bd, scene, nullptr, nullptr, cams, bg, means3D, colors, scales, rotations, opacities, geom, img, binning, radii,
                         out_color, static_cast<cudaStream_t>(stream_));
}

// Checks a GaRasterSets descriptor against the batch (bd checked) and unpacks it into the kernel's form.
static int unpack_sets(const GaRasterBatchDesc *bd, const GaRasterSets *sets, MatteSets &ms)
{
    GA_REQUIRE(sets->K >= 1 && sets->K <= kMaxSets, "bad set count K=%d (1..%d)", (int)sets->K, kMaxSets);
    GA_REQUIRE(sets->first[0] == 0, "sets: first[0] = %d, must be 0", (int)sets->first[0]);
    for (int k = 0; k < sets->K; ++k)
        GA_REQUIRE(sets->first[k + 1] >= sets->first[k], "sets: first[%d] = %d < first[%d] = %d (must not decrease)", k + 1,
                   (int)sets->first[k + 1], k, (int)sets->first[k]);
    GA_REQUIRE(sets->first[sets->K] <= bd->P, "sets: first[K=%d] = %d > P = %d (the sets index the dynamic set)", (int)sets->K,
               (int)sets->first[sets->K], (int)bd->P);
    GA_REQUIRE(sets->mattes != nullptr, "sets: mattes is NULL");
    ms = MatteSets{};
    for (int k = 0; k <= kMaxSets; ++k) ms.first[k] = (uint32_t)sets->first[k < sets->K ? k : sets->K];
    ms.K = sets->K;
    ms.out = sets->mattes;
    return GA_OK;
}

extern "C" int ga_rasterb_forward_mattes(const GaRasterBatchDesc *bd, const GaRasterScene *scene, const GaRasterSets *sets,
                                         const float *cams, const float *bg, const float *means3D, const float *colors, const float *scales,
                                         const float *rotations, const float *opacities, void *geom, void *img, void *binning,
                                         int32_t *radii, float *out_color, void *stream_)
{
    if (int rc = check_batch(bd)) return rc;
    GA_REQUIRE(sets != nullptr, "sets descriptor is NULL");
    MatteSets ms;
    if (int rc = unpack_sets(bd, sets, ms)) return rc;
    if (scene != nullptr && scene->Ps == 0) scene = nullptr;
    return forward_batch(bd, scene, &ms, nullptr, cams, bg, means3D, colors, scales, rotations, opacities, geom, img, binning, radii,
                         out_color, static_cast<cudaStream_t>(stream_));
}

extern "C" int ga_rasterb_forward_depth(const GaRasterBatchDesc *bd, const GaRasterScene *scene, const GaRasterSets *sets, float *depth,
                                        const float *cams, const float *bg, const float *means3D, const float *colors, const float *scales,
                                        const float *rotations, const float *opacities, void *geom, void *img, void *binning,
                                        int32_t *radii, float *out_color, void *stream_)
{
    if (int rc = check_batch(bd)) return rc;
    GA_REQUIRE(depth != nullptr, "depth is NULL");
    MatteSets ms;
    if (sets != nullptr)
        if (int rc = unpack_sets(bd, sets, ms)) return rc;
    if (scene != nullptr && scene->Ps == 0) scene = nullptr;
    return forward_batch(bd, scene, sets ? &ms : nullptr, depth, cams, bg, means3D, colors, scales, rotations, opacities, geom, img,
                         binning, radii, out_color, static_cast<cudaStream_t>(stream_));
}

// The batched backward (bd checked and P > 0 by the caller): dz NULL the colour backward alone, otherwise the depth backward, with
// its state and scratch sizes checked against the batch.  Every check runs before the first launch.
static int backward_batch(const GaRasterBatchDesc *bd, const float *cams, const float *bg, const float *means3D, const float *colors,
                          const float *scales, const float *rotations, const int32_t *radii, const void *geom, const void *img,
                          const void *binning, const float *dL_dout, void *scratch, float *d_means3D, float *d_colors, float *d_scales,
                          float *d_rotations, float *d_opacities, float *d_means2D, cudaStream_t stream, const DepthBwd *dz = nullptr)
{
    GA_REQUIRE(cams && bg && means3D && colors && scales && rotations && radii && geom && img && binning && dL_dout && scratch &&
                   d_means3D && d_colors && d_scales,
               "NULL pointer argument");
    const Dims d = make_dims(bd->B, bd->P, bd->H, bd->W);
    if (dz) {
        if (dz->state.total > dz->state_bytes) {
            set_error("depth state too small: need %zu bytes, have %zu", dz->state.total, dz->state_bytes);
            return GA_ERR_CAPACITY;
        }
        const size_t need = depth_bwd_scratch_bytes((size_t)d.B * d.P);
        if (need > dz->scratch_bytes) {
            set_error("depth backward scratch too small: need %zu bytes, have %zu", need, dz->scratch_bytes);
            return GA_ERR_CAPACITY;
        }
    }
    const BwdArgs a{means3D, colors, scales, rotations, bg, dL_dout, bd->rot_stride, bd->scale_modifier, d_means3D, d_colors, d_scales,
                    d_rotations, d_opacities, d_means2D, bd->antialiasing != 0};
    return launch_backward(d, batch_cams(cams), a, ColorCov{}, radii, carve_geom(const_cast<void *>(geom), (size_t)d.B * d.P),
                           carve_img(const_cast<void *>(img), d), carve_bin(const_cast<void *>(binning), bd->capacity, d), scratch, stream,
                           dz);
}

extern "C" int ga_rasterb_backward(const GaRasterBatchDesc *bd, const float *cams, const float *bg, const float *means3D,
                                   const float *colors, const float *scales, const float *rotations, const int32_t *radii,
                                   const void *geom, const void *img, const void *binning, const float *dL_dout, void *scratch,
                                   float *d_means3D, float *d_colors, float *d_scales, float *d_rotations, float *d_opacities,
                                   float *d_means2D, void *stream_)
{
    if (int rc = check_batch(bd)) return rc;
    if (bd->P == 0) return GA_OK;
    return backward_batch(bd, cams, bg, means3D, colors, scales, rotations, radii, geom, img, binning, dL_dout, scratch, d_means3D, d_colors,
                          d_scales, d_rotations, d_opacities, d_means2D, static_cast<cudaStream_t>(stream_));
}

extern "C" size_t ga_rasterb_depth_state_bytes(int32_t B, int32_t H, int32_t W, int64_t capacity)
{
    return carve_dstate(nullptr, capacity, make_dims(B, 0, H, W)).total;
}
extern "C" size_t ga_rasterb_depth_bwd_scratch_bytes(int32_t B, int32_t P)
{
    return depth_bwd_scratch_bytes((size_t)B * (size_t)(P > 0 ? P : 0));
}

extern "C" int ga_rasterb_forward_depth_train(const GaRasterBatchDesc *bd, float *depth, void *depth_state, size_t depth_state_bytes,
                                              const float *cams, const float *bg, const float *means3D, const float *colors,
                                              const float *scales, const float *rotations, const float *opacities, void *geom, void *img,
                                              void *binning, int32_t *radii, float *out_color, void *stream_)
{
    if (int rc = check_batch(bd)) return rc;
    GA_REQUIRE(depth != nullptr && depth_state != nullptr, "NULL pointer argument");
    const DepthState ds = carve_dstate(depth_state, bd->capacity, make_dims(bd->B, 0, bd->H, bd->W));
    if (ds.total > depth_state_bytes) {
        set_error("depth state too small: need %zu bytes, have %zu", ds.total, depth_state_bytes);
        return GA_ERR_CAPACITY;
    }
    return forward_batch(bd, nullptr, nullptr, depth, cams, bg, means3D, colors, scales, rotations, opacities, geom, img, binning, radii,
                         out_color, static_cast<cudaStream_t>(stream_), &ds);
}

extern "C" int ga_rasterb_backward_depth(const GaRasterBatchDesc *bd, const float *cams, const float *bg, const float *means3D,
                                         const float *colors, const float *scales, const float *rotations, const int32_t *radii,
                                         const void *geom, const void *img, const void *binning, const float *dL_dout,
                                         const float *dL_ddepth, const float *depth, const void *depth_state, size_t depth_state_bytes,
                                         void *scratch, size_t scratch_bytes, float *d_means3D, float *d_colors, float *d_scales,
                                         float *d_rotations, float *d_opacities, float *d_means2D, void *stream_)
{
    if (int rc = check_batch(bd)) return rc;
    if (bd->P == 0) return GA_OK;
    GA_REQUIRE(dL_ddepth && depth && depth_state, "NULL pointer argument");
    const DepthBwd dz{dL_ddepth, depth, carve_dstate(const_cast<void *>(depth_state), bd->capacity, make_dims(bd->B, bd->P, bd->H, bd->W)),
                      depth_state_bytes, scratch_bytes};
    return backward_batch(bd, cams, bg, means3D, colors, scales, rotations, radii, geom, img, binning, dL_dout, scratch, d_means3D, d_colors,
                          d_scales, d_rotations, d_opacities, d_means2D, static_cast<cudaStream_t>(stream_), &dz);
}

extern "C" int ga_raster_views(int32_t B, int32_t P, int32_t H, int32_t W, int64_t capacity, const void *geom, const void *binning,
                               const void *img, GaRasterViews *out)
{
    if (int rc = check_dims(B, P, H, W)) return rc;
    GA_REQUIRE(out, "out is NULL");
    memset(out, 0, sizeof(*out));
    const Dims d = make_dims(B, P, H, W);
    if (geom) {
        GeomViews g = carve_geom(const_cast<void *>(geom), (size_t)B * P);
        out->depth = g.depth; out->xy = reinterpret_cast<const float *>(g.xy);
        out->conic_opacity = reinterpret_cast<const float *>(g.conic_o); out->cov3d = g.cov3d;
        out->tiles_touched = g.tiles; out->rect = reinterpret_cast<const uint16_t *>(g.rect);
    }
    if (binning) {
        BinViews bv = carve_bin(const_cast<void *>(binning), capacity, d);
        out->point_list = bv.point_list;
    }
    if (img) {
        ImgViews iv = carve_img(const_cast<void *>(img), d);
        out->final_T = iv.final_T; out->n_contrib = iv.n_contrib; out->ranges = reinterpret_cast<const uint32_t *>(iv.ranges);
        out->tile_count = iv.count; out->status = iv.status;
    }
    return GA_OK;
}
