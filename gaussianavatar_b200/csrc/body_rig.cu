// Device operators of the body-topology rig (rig.extract_body_rig; DESIGN.md §4): the uniform graph Laplacian the geometry fit
// regularises with, and the push-pull fill that extends a texture from its covered texels to the whole map.  See include/gavatar.h
// for the rules.
//
//   laplacian_kernel     one thread per vertex: y_v = deg_v x_v - sum of x_u over the vertex's CSR row, summed in stored order.
//   pushpull_down_kernel one thread per texel of level l+1: the weighted mean of its (up to four) children at level l that carry
//                        weight, in the fixed order (0,0) (0,1) (1,0) (1,1); weight = the sum of theirs (an exact integer count).
//   pushpull_up_kernel   one thread per texel of level l: a texel without weight takes its parent's (already filled) value.  Level 0
//                        is written to the output, covered texels copied from the input bit for bit.
// Every thread computes its own outputs from its own inputs: no atomics, bit-reproducible.  All fp32 steps are explicitly rounded
// (no contraction), so oracle/body_rig_oracle.py restates them bit for bit.
#include <cstdint>

#include "common.cuh"

namespace ga {
namespace {

constexpr int kBlock = 256;
constexpr int kMaxTexSide = 512;
constexpr int kMaxTexChannels = 4;
constexpr int kMaxLevels = 10;          // 512 -> 256 -> ... -> 1: nine coarse levels

__global__ void __launch_bounds__(kBlock)
laplacian_kernel(int V, const int *__restrict__ offsets, const int *__restrict__ adj, const float *__restrict__ x, float *__restrict__ y)
{
    const int v = blockIdx.x * kBlock + threadIdx.x;
    if (v >= V) return;
    const int b = offsets[v], e = offsets[v + 1];
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int k = b; k < e; ++k) {
        const float *xu = x + 3 * (size_t)adj[k];
        s0 = __fadd_rn(s0, xu[0]); s1 = __fadd_rn(s1, xu[1]); s2 = __fadd_rn(s2, xu[2]);
    }
    const float deg = (float)(e - b);
    const float *xv = x + 3 * (size_t)v;
    float *yv = y + 3 * (size_t)v;
    yv[0] = __fsub_rn(__fmul_rn(deg, xv[0]), s0);
    yv[1] = __fsub_rn(__fmul_rn(deg, xv[1]), s1);
    yv[2] = __fsub_rn(__fmul_rn(deg, xv[2]), s2);
}

// level l (side n, planar values val [C,n,n], weights w [n,n], or mask [n,n] at level 0 with weight 1 per covered texel)
// -> level l+1 (side m)
__global__ void __launch_bounds__(kBlock)
pushpull_down_kernel(int C, int n, int m, const float *__restrict__ val, const float *__restrict__ w, const uint8_t *__restrict__ mask,
                     float *__restrict__ cval, float *__restrict__ cw)
{
    const int t = blockIdx.x * kBlock + threadIdx.x;
    if (t >= m * m) return;
    const int r = t / m, c = t % m;
    float s[kMaxTexChannels] = {0.f, 0.f, 0.f, 0.f};
    float ws = 0.f;
    bool have = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int rr = 2 * r + (k >> 1), cc = 2 * c + (k & 1);
        if (rr >= n || cc >= n) continue;
        const size_t o = (size_t)rr * n + cc;
        const float wk = mask ? (mask[o] ? 1.f : 0.f) : w[o];
        if (!(wk > 0.f)) continue;
#pragma unroll
        for (int ch = 0; ch < kMaxTexChannels; ++ch)
            if (ch < C) {
                const float p = __fmul_rn(wk, val[(size_t)ch * n * n + o]);
                s[ch] = have ? __fadd_rn(s[ch], p) : p;
            }
        ws = have ? __fadd_rn(ws, wk) : wk;
        have = true;
    }
    cw[t] = ws;
#pragma unroll
    for (int ch = 0; ch < kMaxTexChannels; ++ch)
        if (ch < C) cval[(size_t)ch * m * m + t] = have ? __fdiv_rn(s[ch], ws) : 0.f;
}

// level l (side n): texels without weight take the value of their parent at level l+1 (side m, already filled; none when
// pval is NULL: then 0).  Level 0 (mask != NULL) reads the input image and writes the output.
__global__ void __launch_bounds__(kBlock)
pushpull_up_kernel(int C, int n, int m, const float *__restrict__ pval, const float *__restrict__ w, const uint8_t *__restrict__ mask,
                   const float *__restrict__ image, float *__restrict__ val)
{
    const int t = blockIdx.x * kBlock + threadIdx.x;
    if (t >= n * n) return;
    const bool covered = mask ? mask[t] != 0 : w[t] > 0.f;
    const int r = t / n, c = t % n;
    const size_t pt = (size_t)(r >> 1) * m + (c >> 1);
    for (int ch = 0; ch < C; ++ch) {
        const size_t o = (size_t)ch * n * n + t;
        if (covered) {
            if (mask) val[o] = image[o];
        } else {
            val[o] = pval ? pval[(size_t)ch * m * m + pt] : 0.f;
        }
    }
}

struct Pyramid {
    int levels;                          // coarse levels 1..levels
    int side[kMaxLevels + 1];
    float *val[kMaxLevels + 1], *w[kMaxLevels + 1];
    size_t total;
};

Pyramid carve_pyramid(void *p, int S, int C)
{
    Carver cv(p);
    Pyramid py{};
    py.side[0] = S;
    int n = S;
    while (n > 1) {
        n = (n + 1) / 2;
        ++py.levels;
        py.side[py.levels] = n;
        py.val[py.levels] = cv.take<float>((size_t)C * n * n);
        py.w[py.levels] = cv.take<float>((size_t)n * n);
    }
    py.total = cv.used();
    return py;
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_mesh_laplacian(int32_t V, const int32_t *offsets, const int32_t *adj, const float *x, float *y, void *stream_)
{
    GA_REQUIRE(V >= 1 && V <= (1 << 24), "ga_mesh_laplacian: vertex count %d outside [1, 2^24]", V);
    GA_REQUIRE(offsets && adj && x && y, "ga_mesh_laplacian: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("laplacian_kernel", stream);
      laplacian_kernel<<<cdiv(V, kBlock), kBlock, 0, stream>>>(V, offsets, adj, x, y); }
    GA_CHECK_LAUNCH("laplacian_kernel");
    return GA_OK;
}

extern "C" size_t ga_texture_pushpull_workspace_bytes(int32_t S, int32_t C)
{
    if (S < 1 || S > kMaxTexSide || C < 1 || C > kMaxTexChannels) return 0;
    return carve_pyramid(nullptr, S, C).total;
}

extern "C" int ga_texture_pushpull(int32_t S, int32_t C, const float *image, const uint8_t *mask, void *workspace, size_t workspace_bytes,
                                   float *out, void *stream_)
{
    GA_REQUIRE(S >= 1 && S <= kMaxTexSide, "ga_texture_pushpull: map size %d outside [1, %d]", S, kMaxTexSide);
    GA_REQUIRE(C >= 1 && C <= kMaxTexChannels, "ga_texture_pushpull: %d channels outside [1, %d]", C, kMaxTexChannels);
    GA_REQUIRE(image && mask && out, "ga_texture_pushpull: NULL pointer argument");
    const size_t need = carve_pyramid(nullptr, S, C).total;
    GA_REQUIRE(need == 0 || workspace, "ga_texture_pushpull: NULL pointer argument");
    GA_REQUIRE(workspace_bytes >= need, "ga_texture_pushpull: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    GA_REQUIRE(reinterpret_cast<uintptr_t>(workspace) % kAlign == 0, "ga_texture_pushpull: workspace must be %zu-byte aligned", kAlign);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const Pyramid py = carve_pyramid(workspace, S, C);
    for (int l = 0; l < py.levels; ++l) {
        const int n = py.side[l], m = py.side[l + 1];
        { ProfScope _ps("pushpull_down_kernel", stream);
          pushpull_down_kernel<<<cdiv((long long)m * m, kBlock), kBlock, 0, stream>>>(C, n, m, l ? py.val[l] : image, py.w[l],
                                                                                       l ? nullptr : mask, py.val[l + 1], py.w[l + 1]); }
        GA_CHECK_LAUNCH("pushpull_down_kernel");
    }
    // the coarsest level is complete as the down pass left it (its one texel is 0 when nothing is covered)
    for (int l = py.levels > 0 ? py.levels - 1 : 0; l >= 0; --l) {
        const int n = py.side[l], m = l < py.levels ? py.side[l + 1] : 1;
        const float *pval = l < py.levels ? py.val[l + 1] : nullptr;
        { ProfScope _ps("pushpull_up_kernel", stream);
          pushpull_up_kernel<<<cdiv((long long)n * n, kBlock), kBlock, 0, stream>>>(C, n, m, pval, py.w[l], l ? nullptr : mask,
                                                                                     image, l ? py.val[l] : out); }
        GA_CHECK_LAUNCH("pushpull_up_kernel");
    }
    return GA_OK;
}
