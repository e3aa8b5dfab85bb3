// Skin-weight transfer from an avatar's canonical Gaussians to the vertices of a mesh extracted from them (DESIGN.md §2, defined
// here).  See include/gavatar.h for the rule.
//
//   skin_weights_kernel  one thread per vertex, n-body style: the block stages tiles of kTile means through shared memory and every
//                        thread scans each tile for its vertex's k nearest means, kept sorted in registers (distance, then index).
//                        Then it blends the neighbours' skinning rows in fp64 in neighbour order and keeps the K heaviest joints,
//                        also in registers.  A vertex's result depends on nothing but its own inputs: no atomics, no reductions
//                        across threads, so the output is bit-reproducible and independent of the launch split.
#include <cstdint>

#include "common.cuh"

namespace ga {
namespace {

constexpr int kMaxNeighbours = 16;      // k
constexpr int kMaxInfluences = 8;       // K
constexpr int kMaxLd = 256;
constexpr int kBlock = 128;
constexpr int kTile = 512;              // means per shared-memory tile
constexpr double kEps2 = 1e-6;          // eps^2, eps = 1e-3 world units

// The squared distance, one fixed fp32 expression without contraction: ((dx dx + dy dy) + dz dz), d = mean - vertex.
__device__ __forceinline__ float dist2(float4 m, float vx, float vy, float vz)
{
    const float dx = __fsub_rn(m.x, vx), dy = __fsub_rn(m.y, vy), dz = __fsub_rn(m.z, vz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__global__ void __launch_bounds__(kBlock, 4)
skin_weights_kernel(int V, int N, int J, int ld, int k, int K, const float *__restrict__ verts, const float *__restrict__ means,
                    const float *__restrict__ lbs, uint8_t *__restrict__ joints, float *__restrict__ weights)
{
    __shared__ float4 tile[kTile];
    const int v = blockIdx.x * kBlock + threadIdx.x;
    const int vc = v < V ? v : V - 1;
    const float vx = verts[3 * (size_t)vc], vy = verts[3 * (size_t)vc + 1], vz = verts[3 * (size_t)vc + 2];

    // the k nearest in slots 0..k-1, worst first: descending by (distance, index), so the one to evict is always slot 0 and every
    // index into the list is a compile-time constant (registers only)
    float nd[kMaxNeighbours];
    int ni[kMaxNeighbours];
#pragma unroll
    for (int s = 0; s < kMaxNeighbours; ++s) { nd[s] = __int_as_float(0x7f800000); ni[s] = 0; }
    for (int base = 0; base < N; base += kTile) {
        const int n = min(kTile, N - base);
        __syncthreads();
        for (int t = threadIdx.x; t < n; t += kBlock) {
            const float *p = means + 3 * ((size_t)base + t);
            tile[t] = make_float4(p[0], p[1], p[2], 0.f);
        }
        __syncthreads();
#pragma unroll 4
        for (int t = 0; t < n; ++t) {
            const float d = dist2(tile[t], vx, vy, vz);
            if (d < nd[0]) {               // strict: the means come in index order, so an equal distance keeps the lower index
                const int id = base + t;
                bool placed = false;
#pragma unroll
                for (int s = 0; s < kMaxNeighbours; ++s) {
                    if (!placed && s < k) {
                        if (s + 1 < kMaxNeighbours && s + 1 < k && nd[s + 1] > d) { nd[s] = nd[s + 1]; ni[s] = ni[s + 1]; }
                        else { nd[s] = d; ni[s] = id; placed = true; }
                    }
                }
            }
        }
    }
    if (v >= V) return;

    // neighbour order (nearest first) is slot k-1 down to 0
    double c[kMaxNeighbours], den = 0.0;
#pragma unroll
    for (int s = kMaxNeighbours - 1; s >= 0; --s) {
        c[s] = 1.0 / __dadd_rn((double)nd[s], kEps2);
        if (s < k) den = __dadd_rn(den, c[s]);
    }
    // the K heaviest joints of positive blended weight in slots 0..K-1, lightest first: ascending by (weight, -index); empty slots
    // hold weight 0
    double sw[kMaxInfluences];
    int sj[kMaxInfluences];
#pragma unroll
    for (int s = 0; s < kMaxInfluences; ++s) { sw[s] = 0.0; sj[s] = 0; }
    for (int j = 0; j < J; ++j) {
        double num = 0.0;
#pragma unroll
        for (int s = kMaxNeighbours - 1; s >= 0; --s)
            if (s < k) num = __dadd_rn(num, __dmul_rn(c[s], (double)__ldg(lbs + (size_t)ni[s] * ld + j)));
        const double w = num / den;
        if (w > sw[0]) {                   // strict: the joints come in index order, so an equal weight keeps the lower joint
            bool placed = false;
#pragma unroll
            for (int s = 0; s < kMaxInfluences; ++s) {
                if (!placed && s < K) {
                    if (s + 1 < kMaxInfluences && s + 1 < K && sw[s + 1] < w) { sw[s] = sw[s + 1]; sj[s] = sj[s + 1]; }
                    else { sw[s] = w; sj[s] = j; placed = true; }
                }
            }
        }
    }
    // written heaviest first: output slot K-1-s
    double sum = 0.0;
#pragma unroll
    for (int s = kMaxInfluences - 1; s >= 0; --s)
        if (s < K) sum = __dadd_rn(sum, sw[s]);
    uint8_t *jo = joints + (size_t)v * K;
    float *wo = weights + (size_t)v * K;
#pragma unroll
    for (int s = 0; s < kMaxInfluences; ++s) {
        if (s < K) {
            const int o = K - 1 - s;
            if (sum > 0.0) {
                jo[o] = (uint8_t)sj[s];
                wo[o] = (float)(sw[s] / sum);
            } else {                       // no joint carries weight: bind to the root
                jo[o] = 0;
                wo[o] = o == 0 ? 1.f : 0.f;
            }
        }
    }
}

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_skin_weights(int32_t V, int32_t N, int32_t J, int32_t ld, int32_t k, int32_t K, const float *verts, const float *means,
                               const float *lbs, uint8_t *joints, float *weights, void *stream_)
{
    GA_REQUIRE(V >= 1 && N >= 1, "ga_skin_weights: %d vertices and %d Gaussians must both be >= 1", V, N);
    GA_REQUIRE(ld >= 1 && ld <= kMaxLd && J >= 1 && J <= ld, "ga_skin_weights: J = %d, ld = %d: need 1 <= J <= ld <= %d", J, ld, kMaxLd);
    GA_REQUIRE(k >= 1 && k <= kMaxNeighbours && k <= N, "ga_skin_weights: k = %d outside [1, min(%d, N = %d)]", k, kMaxNeighbours, N);
    GA_REQUIRE(K >= 1 && K <= kMaxInfluences && K <= J, "ga_skin_weights: K = %d outside [1, min(%d, J = %d)]", K, kMaxInfluences, J);
    GA_REQUIRE(verts && means && lbs && joints && weights, "ga_skin_weights: NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    { ProfScope _ps("skin_weights_kernel", stream);
      skin_weights_kernel<<<cdiv(V, kBlock), kBlock, 0, stream>>>(V, N, J, ld, k, K, verts, means, lbs, joints, weights); }
    GA_CHECK_LAUNCH("skin_weights_kernel");
    return GA_OK;
}
