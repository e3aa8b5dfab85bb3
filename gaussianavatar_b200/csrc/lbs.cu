// Fused Gaussian linear-blend skinning + per-Gaussian attribute assembly, forward + backward.
//
// Replaces /root/reference model/avatar_model.py:308-326 (and the identical blocks at :404-424, :499-517, :594-612):
//   pred_res * 0.02 -> mask-select -> + query_points -> einsum('bnj,bjxy->bnxy') -> einsum('bnxy,bny->bnx') + t,
//   the iteration<1000 scale ramp, the mask-selects of scales / colours and `repeat(1,1,3)`.
// The reference materialises pt_mats [B,N,4,4] and runs ~10 kernels + 3 nonzero() host syncs; here one persistent
// kernel streams the [N,24] skinning-weight table through shared memory with 1-D TMA bulk copies
// (cp.async.bulk + mbarrier, two stages), reads it ONCE for all B frames of the step, and writes means3D / scales /
// colours directly in the rasterizer's layout.  Decoder outputs arrive pixel-major packed [S*S, 8] =
// (res.xyz, scale, rgb, pad); `vidx[n]` is the flat UV index of the n-th valid pixel (order of the boolean mask).
//
// The kernel is a template over the body model: kJ joints, kLd floats per weight row (a multiple of 4: 16-byte rows for the TMA
// copy and the float4 row reads).  SMPL is (24, 24): ~71 KB of shared memory, two CTAs per SM, the weights held in registers.
// SMPL-X is (55, 56), the table padded with a zero column: ~149 KB, one CTA per SM, the weights read from shared memory where
// they are used (55 more live registers would spill).
//
// kExposure adds each frame's colour transform c' = A c + t (the [A | t] row of a per-training-frame table, gathered through
// pose_idx on the device) to the colours the kernel writes, and in the backward the decoder colour gradient A^T g and the table's
// gradient: per CTA and frame slot the 12 sums of g (x) [c, 1], one more row of the block-level product, written to a workspace that
// lbs_exposure_reduce_kernel adds up in a fixed order (DESIGN.md §4).  The kernels without it are unchanged.
#include <type_traits>

#include "common.cuh"

namespace ga {
namespace {

constexpr int kTileN = 256;     // Gaussians per tile == threads per CTA
constexpr int kMaxFrames = 8;
constexpr int kStages = 2;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (bytes % 16 == 0, 16-B aligned addresses)
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

template <int kJ, int kLd>
struct alignas(128) LbsSmem {
    float w[kStages][kTileN * kLd];       // 2 x 24 KB (SMPL) / 2 x 56 KB (SMPL-X) skinning-weight tiles (TMA destination)
    float C[kMaxFrames][kJ * 12];         // cano2live 3x4 per joint, all frames of the step
    float x[kTileN][13];                  // backward: per-Gaussian [g (x) c | g], padded against bank conflicts
    uint64_t full[kStages];
};

// the exposure variant appends its arrays, so that the layout above stays as it is
template <int kJ, int kLd>
struct alignas(128) LbsSmemExp : LbsSmem<kJ, kLd> {
    float E[kMaxFrames][12];              // [A | t] of every frame of the step (row-major 3x4)
    float xe[kTileN][13];                 // backward: per-Gaussian g_colour (x) [c | 1]
    float eacc[kMaxFrames][12];           // backward: this CTA's exposure sums, each element owned by one thread
};

template <bool kExposure, int kJ, int kLd>
using LbsSmemT = std::conditional_t<kExposure, LbsSmemExp<kJ, kLd>, LbsSmem<kJ, kLd>>;

template <bool kBackward, int kJ, int kLd, bool kExposure = false>
__global__ void __launch_bounds__(kTileN)
lbs_kernel(int N, int B, float scale_mul, long long dec_stride /*floats between two frames' decoder outputs; 0: one output shared by all*/,
           const float *__restrict__ dec /*[S*S,8] or [B][S*S,8]*/, const int32_t *__restrict__ vidx,
           const float *__restrict__ q /*[N,3]*/, const float *__restrict__ w /*[N,kLd]*/,
           const float *__restrict__ Cg /*[B,kJ,12]*/,
           // forward outputs
           float *__restrict__ means, float *__restrict__ scales3, float *__restrict__ colors,
           // backward inputs / outputs
           const float *__restrict__ d_means, const float *__restrict__ d_scales3, const float *__restrict__ d_colors,
           float *__restrict__ d_dec /*[S*S,8], pre-zeroed*/, float *__restrict__ dC /*[B,kJ,12], pre-zeroed*/,
           // kExposure: the [F,12] table, the frames' rows in it and (backward) the per-CTA partials [gridDim.x][kMaxFrames][12]
           int F, const float *__restrict__ Et, const int32_t *__restrict__ pidx, float *__restrict__ dE_part)
{
    static_assert(kLd % 4 == 0 && kLd >= kJ, "weight rows are whole float4s");
    constexpr bool kRegW = kJ <= 24;           // weights of this thread's Gaussian kept in registers across the frames
    constexpr int kOuts = kJ * 12 + (kExposure ? 12 : 0);   // dC, then the exposure sums
    constexpr int kOut = (kOuts + kTileN - 1) / kTileN;    // outputs per thread per frame
    extern __shared__ __align__(128) unsigned char smem_raw[];
    LbsSmemT<kExposure, kJ, kLd> &sm = *reinterpret_cast<LbsSmemT<kExposure, kJ, kLd> *>(smem_raw);
    const int tid = threadIdx.x;
    const int tiles = (N + kTileN - 1) / kTileN;

    for (int i = tid; i < B * kJ * 12; i += kTileN) sm.C[i / (kJ * 12)][i % (kJ * 12)] = Cg[i];
    if constexpr (kExposure) {   // a frame whose row is outside the table gets NaN colours: the error shows in the image, not as a stray read
        for (int i = tid; i < B * 12; i += kTileN) {
            const int f = pidx[i / 12];
            sm.E[i / 12][i % 12] = (f >= 0 && f < F) ? Et[(size_t)f * 12 + i % 12] : __int_as_float(0x7fffffff);
        }
        if (kBackward)
            for (int i = tid; i < kMaxFrames * 12; i += kTileN) sm.eacc[i / 12][i % 12] = 0.f;
    }
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(&sm.full[s], 1);
        fence_barrier_init();
    }
    __syncthreads();

    auto issue = [&](int tile, int stage) {
        const int n0 = tile * kTileN;
        const uint32_t bytes = (uint32_t)min(kTileN, N - n0) * kLd * sizeof(float);
        mbar_expect_tx(&sm.full[stage], bytes);
        tma_load_1d(sm.w[stage], w + (size_t)n0 * kLd, bytes, &sm.full[stage]);
    };
    int tile = blockIdx.x;
    if (tid == 0 && tile < tiles) issue(tile, 0);

    float acc[kMaxFrames][kOut];   // backward: this thread's dC outputs (o = tid, tid + 256, ...), per frame
    if (kBackward) {
#pragma unroll
        for (int b = 0; b < kMaxFrames; ++b)
#pragma unroll
            for (int h = 0; h < kOut; ++h) acc[b][h] = 0.f;
    }

    int it = 0;
    for (; tile < tiles; tile += gridDim.x, ++it) {
        const int stage = it & 1;
        const int next = tile + gridDim.x;
        if (tid == 0 && next < tiles) issue(next, stage ^ 1);   // the other stage was fully consumed last iteration
        mbar_wait(&sm.full[stage], (it >> 1) & 1);

        const int n = tile * kTileN + tid;
        const bool valid = n < N;
        const float *wr = sm.w[stage] + tid * kLd;
        float cx = 0.f, cy = 0.f, cz = 0.f, sc = 0.f, r = 0.f, g = 0.f, bl = 0.f;
        int vi = 0;
        if (valid) {
            vi = vidx[n];
            const float4 o0 = *reinterpret_cast<const float4 *>(dec + (size_t)vi * 8);
            const float4 o1 = *reinterpret_cast<const float4 *>(dec + (size_t)vi * 8 + 4);
            cx = q[(size_t)n * 3] + 0.02f * o0.x; cy = q[(size_t)n * 3 + 1] + 0.02f * o0.y; cz = q[(size_t)n * 3 + 2] + 0.02f * o0.z;
            sc = o0.w * scale_mul; r = o1.x; g = o1.y; bl = o1.z;
        }
        float wv[kRegW ? kJ : 1];
        if constexpr (kRegW) {
            if (valid) {
#pragma unroll
                for (int k = 0; k < kJ / 4; ++k) {
                    const float4 t = *reinterpret_cast<const float4 *>(wr + 4 * k);
                    wv[4 * k] = t.x; wv[4 * k + 1] = t.y; wv[4 * k + 2] = t.z; wv[4 * k + 3] = t.w;
                }
            } else {
#pragma unroll
                for (int k = 0; k < kJ; ++k) wv[k] = 0.f;
            }
        }
        float dcx = 0.f, dcy = 0.f, dcz = 0.f, dsc = 0.f, dr = 0.f, dg = 0.f, dbl = 0.f;
        for (int b = 0; b < B; ++b) {
            if (dec_stride && valid) {          // stage 2: every frame has its own decoder output
                const float *db = dec + (size_t)b * dec_stride + (size_t)vi * 8;
                const float4 o0 = *reinterpret_cast<const float4 *>(db), o1 = *reinterpret_cast<const float4 *>(db + 4);
                cx = q[(size_t)n * 3] + 0.02f * o0.x; cy = q[(size_t)n * 3 + 1] + 0.02f * o0.y; cz = q[(size_t)n * 3 + 2] + 0.02f * o0.z;
                sc = o0.w * scale_mul; r = o1.x; g = o1.y; bl = o1.z;
            }
            float M[12];
#pragma unroll
            for (int e = 0; e < 12; ++e) M[e] = 0.f;
            if constexpr (kRegW) {
#pragma unroll
                for (int j = 0; j < kJ; ++j) {
                    const float wj = wv[j];
#pragma unroll
                    for (int e = 0; e < 12; ++e) M[e] = fmaf(wj, sm.C[b][j * 12 + e], M[e]);
                }
            } else if (valid) {   // invalid rows keep M = 0 (their smem row is stale)
#pragma unroll
                for (int k = 0; k < kLd / 4; ++k) {
                    const float4 t = *reinterpret_cast<const float4 *>(wr + 4 * k);
                    const float wq[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int j = 4 * k + i;
                        if (j < kJ) {
#pragma unroll
                            for (int e = 0; e < 12; ++e) M[e] = fmaf(wq[i], sm.C[b][j * 12 + e], M[e]);
                        }
                    }
                }
            }
            const size_t o = ((size_t)b * N + n) * 3;
            if (!kBackward) {
                if (valid) {
                    means[o] = M[0] * cx + M[1] * cy + M[2] * cz + M[3];
                    means[o + 1] = M[4] * cx + M[5] * cy + M[6] * cz + M[7];
                    means[o + 2] = M[8] * cx + M[9] * cy + M[10] * cz + M[11];
                    scales3[o] = sc; scales3[o + 1] = sc; scales3[o + 2] = sc;
                    if constexpr (kExposure) {
                        const float *E = sm.E[b];
                        colors[o] = fmaf(E[0], r, fmaf(E[1], g, fmaf(E[2], bl, E[3])));
                        colors[o + 1] = fmaf(E[4], r, fmaf(E[5], g, fmaf(E[6], bl, E[7])));
                        colors[o + 2] = fmaf(E[8], r, fmaf(E[9], g, fmaf(E[10], bl, E[11])));
                    } else {
                        colors[o] = r; colors[o + 1] = g; colors[o + 2] = bl;
                    }
                }
            } else {
                float g0 = 0.f, g1 = 0.f, g2 = 0.f;
                float h0 = 0.f, h1 = 0.f, h2 = 0.f;     // kExposure: the transformed colours' gradient
                if (valid) {
                    g0 = d_means[o]; g1 = d_means[o + 1]; g2 = d_means[o + 2];
                    dcx += M[0] * g0 + M[4] * g1 + M[8] * g2;
                    dcy += M[1] * g0 + M[5] * g1 + M[9] * g2;
                    dcz += M[2] * g0 + M[6] * g1 + M[10] * g2;
                    dsc += d_scales3[o] + d_scales3[o + 1] + d_scales3[o + 2];
                    if constexpr (kExposure) {           // A^T g
                        const float *E = sm.E[b];
                        h0 = d_colors[o]; h1 = d_colors[o + 1]; h2 = d_colors[o + 2];
                        dr += fmaf(E[0], h0, fmaf(E[4], h1, E[8] * h2));
                        dg += fmaf(E[1], h0, fmaf(E[5], h1, E[9] * h2));
                        dbl += fmaf(E[2], h0, fmaf(E[6], h1, E[10] * h2));
                    } else {
                        dr += d_colors[o]; dg += d_colors[o + 1]; dbl += d_colors[o + 2];
                    }
                }
                // dC[b][j][r*4 + c] += w[n][j] * (c < 3 ? g_r * c_c : g_r): block-level (kJ x 256) x (256 x 12) product
                __syncthreads();
                float *xr = sm.x[tid];
                xr[0] = g0 * cx; xr[1] = g0 * cy; xr[2] = g0 * cz; xr[3] = g0;
                xr[4] = g1 * cx; xr[5] = g1 * cy; xr[6] = g1 * cz; xr[7] = g1;
                xr[8] = g2 * cx; xr[9] = g2 * cy; xr[10] = g2 * cz; xr[11] = g2;
                if constexpr (kExposure) {           // dE[r*4 + k] += g_r * [c | 1]_k, c the decoder colour of this frame
                    float *xq = sm.xe[tid];
                    xq[0] = h0 * r; xq[1] = h0 * g; xq[2] = h0 * bl; xq[3] = h0;
                    xq[4] = h1 * r; xq[5] = h1 * g; xq[6] = h1 * bl; xq[7] = h1;
                    xq[8] = h2 * r; xq[9] = h2 * g; xq[10] = h2 * bl; xq[11] = h2;
                }
                __syncthreads();
                const float *ws = sm.w[stage];
#pragma unroll
                for (int h = 0; h < kOut; ++h) {
                    const int oidx = tid + h * kTileN;
                    if (oidx < kJ * 12) {
                        const int j = oidx / 12, e = oidx % 12;
                        float t = 0.f;
                        const int rows = min(kTileN, N - tile * kTileN);
                        for (int m = 0; m < rows; ++m) t = fmaf(ws[m * kLd + j], sm.x[m][e], t);
                        acc[b][h] += t;
                    } else if constexpr (kExposure) {
                        if (oidx < kOuts) {          // threads past dC's: the tile's exposure sums, in row order
                            const int e = oidx - kJ * 12;
                            float t = 0.f;
                            const int rows = min(kTileN, N - tile * kTileN);
                            for (int m = 0; m < rows; ++m) t += sm.xe[m][e];
                            sm.eacc[b][e] += t;
                        }
                    }
                }
                if (dec_stride) {               // per-frame decoder output: this frame's gradient goes to this frame's rows
                    if (valid) {
                        float *db = d_dec + (size_t)b * dec_stride + (size_t)vi * 8;
                        *reinterpret_cast<float4 *>(db) = make_float4(0.02f * dcx, 0.02f * dcy, 0.02f * dcz, scale_mul * dsc);
                        *reinterpret_cast<float4 *>(db + 4) = make_float4(dr, dg, dbl, 0.f);
                    }
                    dcx = dcy = dcz = dsc = dr = dg = dbl = 0.f;
                }
            }
        }
        if (kBackward && valid && !dec_stride) {
            float4 o0 = make_float4(0.02f * dcx, 0.02f * dcy, 0.02f * dcz, scale_mul * dsc);
            float4 o1 = make_float4(dr, dg, dbl, 0.f);
            *reinterpret_cast<float4 *>(d_dec + (size_t)vi * 8) = o0;
            *reinterpret_cast<float4 *>(d_dec + (size_t)vi * 8 + 4) = o1;
        }
        __syncthreads();   // every thread is done with sm.w[stage] before it is refilled two iterations later
    }
    if (kBackward) {
        for (int b = 0; b < B; ++b)
#pragma unroll
            for (int h = 0; h < kOut; ++h) {
                const int oidx = tid + h * kTileN;
                if (oidx < kJ * 12 && acc[b][h] != 0.f) atomicAdd(&dC[(size_t)b * kJ * 12 + oidx], acc[b][h]);
            }
        if constexpr (kExposure)   // the tile loop ended on a barrier: every thread's sums are visible
            for (int i = tid; i < B * 12; i += kTileN) dE_part[((size_t)blockIdx.x * kMaxFrames + i / 12) * 12 + i % 12] = sm.eacc[i / 12][i % 12];
    }
}

// dE[f][e] = sum over the slots b with pidx[b] == f, in slot order, of slot b's per-CTA partials; 0 for rows no slot touched and
// for row 0, the gauge anchor.  One warp per table element: lane l adds the partials of CTAs l, l + 32, ... in order, then a fixed
// xor-shuffle tree adds the lanes.  No atomics: a replay gives the same bits.
constexpr int kReduceWarps = 8;
__global__ void __launch_bounds__(32 * kReduceWarps)
lbs_exposure_reduce_kernel(int F, int B, int ctas, const int32_t *__restrict__ pidx, const float *__restrict__ part, float *__restrict__ dE)
{
    const int i = blockIdx.x * kReduceWarps + (int)(threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= F * 12) return;                      // whole warps leave together
    const int f = i / 12, e = i % 12;
    float s = 0.f;
    if (f > 0) {
        for (int b = 0; b < B; ++b) {
            if (pidx[b] != f) continue;           // the same branch for every lane of the warp
            float t = 0.f;
            for (int c = lane; c < ctas; c += 32) t += part[((size_t)c * kMaxFrames + b) * 12 + e];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            s += t;
        }
    }
    if (lane == 0) dE[i] = s;
}

// Persistent grid: as many CTAs as fit on the SMs at once, capped by the tile count.  SMPL (~71 KB, ~85 KB with the exposure) fits
// two per SM, SMPL-X (~149 KB, ~163 KB) one.
template <int kJ, int kLd, bool kExposure = false>
int launch_cfg(int N)
{
    constexpr int per_sm = sizeof(LbsSmemT<kExposure, kJ, kLd>) <= 113 * 1024 ? 2 : 1;
    const int tiles = cdiv(N, kTileN);
    return tiles < per_sm * kNumSMs ? tiles : per_sm * kNumSMs;
}

// Exposure arguments of a launch: the table [F,12], the frames' rows pidx [B] and the backward's per-CTA partials
struct ExposureArgs {
    int F = 0;
    const float *table = nullptr;
    const int32_t *pidx = nullptr;
    float *partials = nullptr;
};

template <int kJ, int kLd, bool kExposure>
int set_smem_attrs()
{
    static PerDeviceOnce attr_set;
    if (attr_set.first()) {
        constexpr int bytes = (int)sizeof(LbsSmemT<kExposure, kJ, kLd>);
        GA_CHECK_CUDA(cudaFuncSetAttribute(lbs_kernel<false, kJ, kLd, kExposure>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        GA_CHECK_CUDA(cudaFuncSetAttribute(lbs_kernel<true, kJ, kLd, kExposure>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    }
    return GA_OK;
}

template <int kJ, int kLd, bool kExposure = false>
int lbs_forward(int N, int B, float scale_mul, int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index,
                const float *query_points, const float *query_lbs, const float *cano2live, float *means3D, float *scales3, float *colors,
                cudaStream_t stream, const char *name, ExposureArgs ex = {})
{
    if (const int rc = set_smem_attrs<kJ, kLd, kExposure>()) return rc;
    { ProfScope _ps(name, stream); lbs_kernel<false, kJ, kLd, kExposure><<<launch_cfg<kJ, kLd, kExposure>(N), kTileN,
        sizeof(LbsSmemT<kExposure, kJ, kLd>), stream>>>(
        N, B, scale_mul, (long long)dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, means3D, scales3, colors, nullptr, nullptr,
        nullptr, nullptr, nullptr, ex.F, ex.table, ex.pidx, nullptr); }
    GA_CHECK_LAUNCH(name);
    return GA_OK;
}

template <int kJ, int kLd, bool kExposure = false>
int lbs_backward(int N, int B, float scale_mul, int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index,
                 const float *query_points, const float *query_lbs, const float *cano2live, const float *d_means3D, const float *d_scales3,
                 const float *d_colors, float *d_dec_out, float *d_cano2live, cudaStream_t stream, const char *name, ExposureArgs ex = {})
{
    if (const int rc = set_smem_attrs<kJ, kLd, kExposure>()) return rc;
    { ProfScope _ps(name, stream); lbs_kernel<true, kJ, kLd, kExposure><<<launch_cfg<kJ, kLd, kExposure>(N), kTileN,
        sizeof(LbsSmemT<kExposure, kJ, kLd>), stream>>>(N, B, scale_mul,
        (long long)dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, nullptr, nullptr, nullptr,
        d_means3D, d_scales3, d_colors, d_dec_out, d_cano2live, ex.F, ex.table, ex.pidx, ex.partials); }
    GA_CHECK_LAUNCH(name);
    return GA_OK;
}

// CTAs of the exposure backward (one partial row block each); 0 for a layout that is not built
int exposure_ctas(int N, int num_joints)
{
    if (num_joints == 24) return launch_cfg<24, 24, true>(N);
    if (num_joints == 55) return launch_cfg<55, 56, true>(N);
    return 0;
}

// The built (joints, row stride) layouts.  Any other pair that passes the ABI's checks is refused with a message naming these.
bool built_layout(int num_joints, int lbs_ld) { return (num_joints == 24 && lbs_ld == 24) || (num_joints == 55 && lbs_ld == 56); }

}  // namespace
}  // namespace ga

using namespace ga;

extern "C" int ga_lbs_forward_ex(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, float scale_mul, int64_t dec_frame_stride,
                                 const float *dec_out, const int32_t *valid_index, const float *query_points, const float *query_lbs,
                                 const float *cano2live, float *means3D, float *scales3, float *colors, void *stream_)
{
    GA_REQUIRE(N >= 0 && B >= 1 && B <= kMaxFrames, "bad LBS dims N=%d B=%d (B <= %d)", N, B, kMaxFrames);
    GA_REQUIRE(num_joints == 24 || num_joints == 55, "num_joints %d: 24 (SMPL) or 55 (SMPL-X)", num_joints);
    GA_REQUIRE(lbs_ld % 4 == 0 && lbs_ld >= num_joints, "lbs_ld %d: a multiple of 4 and >= num_joints %d", lbs_ld, num_joints);
    GA_REQUIRE(built_layout(num_joints, lbs_ld), "lbs_ld %d for %d joints is not built (24 joints: 24; 55 joints: 56)", lbs_ld, num_joints);
    if (N == 0) return GA_OK;
    GA_REQUIRE(dec_out && valid_index && query_points && query_lbs && cano2live && means3D && scales3 && colors, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (num_joints == 24)
        return lbs_forward<24, 24>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, means3D, scales3,
                                   colors, stream, "lbs_kernel<fwd>");
    return lbs_forward<55, 56>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, means3D, scales3,
                               colors, stream, "lbs_kernel<fwd,55>");
}

extern "C" int ga_lbs_backward_ex(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, int32_t num_pixels, float scale_mul,
                                  int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index, const float *query_points,
                                  const float *query_lbs, const float *cano2live, const float *d_means3D, const float *d_scales3,
                                  const float *d_colors, float *d_dec_out, float *d_cano2live, void *stream_)
{
    GA_REQUIRE(N >= 0 && B >= 1 && B <= kMaxFrames && num_pixels >= N, "bad LBS dims N=%d B=%d pixels=%d", N, B, num_pixels);
    GA_REQUIRE(num_joints == 24 || num_joints == 55, "num_joints %d: 24 (SMPL) or 55 (SMPL-X)", num_joints);
    GA_REQUIRE(lbs_ld % 4 == 0 && lbs_ld >= num_joints, "lbs_ld %d: a multiple of 4 and >= num_joints %d", lbs_ld, num_joints);
    GA_REQUIRE(built_layout(num_joints, lbs_ld), "lbs_ld %d for %d joints is not built (24 joints: 24; 55 joints: 56)", lbs_ld, num_joints);
    GA_REQUIRE(d_dec_out && d_cano2live, "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    GA_CHECK_CUDA(cudaMemsetAsync(d_dec_out, 0, sizeof(float) * 8 * (size_t)num_pixels, stream));
    GA_CHECK_CUDA(cudaMemsetAsync(d_cano2live, 0, sizeof(float) * num_joints * 12 * (size_t)B, stream));
    if (N == 0) return GA_OK;
    GA_REQUIRE(dec_out && valid_index && query_points && query_lbs && cano2live && d_means3D && d_scales3 && d_colors, "NULL pointer argument");
    if (num_joints == 24)
        return lbs_backward<24, 24>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, d_means3D,
                                    d_scales3, d_colors, d_dec_out, d_cano2live, stream, "lbs_kernel<bwd>");
    return lbs_backward<55, 56>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, d_means3D,
                                d_scales3, d_colors, d_dec_out, d_cano2live, stream, "lbs_kernel<bwd,55>");
}

extern "C" size_t ga_lbs_exposure_workspace_bytes(int32_t N, int32_t num_joints)
{
    return N > 0 ? sizeof(float) * 12 * kMaxFrames * (size_t)exposure_ctas(N, num_joints) : 0;
}

extern "C" int ga_lbs_forward_exposure(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, float scale_mul, int64_t dec_frame_stride,
                                       const float *dec_out, const int32_t *valid_index, const float *query_points, const float *query_lbs,
                                       const float *cano2live, int32_t num_exposures, const float *exposure, const int32_t *pose_idx,
                                       float *means3D, float *scales3, float *colors, void *stream_)
{
    GA_REQUIRE(N >= 0 && B >= 1 && B <= kMaxFrames, "bad LBS dims N=%d B=%d (B <= %d)", N, B, kMaxFrames);
    GA_REQUIRE(num_joints == 24 || num_joints == 55, "num_joints %d: 24 (SMPL) or 55 (SMPL-X)", num_joints);
    GA_REQUIRE(lbs_ld % 4 == 0 && lbs_ld >= num_joints, "lbs_ld %d: a multiple of 4 and >= num_joints %d", lbs_ld, num_joints);
    GA_REQUIRE(built_layout(num_joints, lbs_ld), "lbs_ld %d for %d joints is not built (24 joints: 24; 55 joints: 56)", lbs_ld, num_joints);
    GA_REQUIRE(num_exposures >= 1, "num_exposures %d: the exposure table needs at least one row", num_exposures);
    if (N == 0) return GA_OK;
    GA_REQUIRE(dec_out && valid_index && query_points && query_lbs && cano2live && exposure && pose_idx && means3D && scales3 && colors,
               "NULL pointer argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    ExposureArgs ex;
    ex.F = num_exposures; ex.table = exposure; ex.pidx = pose_idx;
    if (num_joints == 24)
        return lbs_forward<24, 24, true>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, means3D,
                                         scales3, colors, stream, "lbs_kernel<fwd,exposure>", ex);
    return lbs_forward<55, 56, true>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, means3D,
                                     scales3, colors, stream, "lbs_kernel<fwd,55,exposure>", ex);
}

extern "C" int ga_lbs_backward_exposure(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, int32_t num_pixels, float scale_mul,
                                        int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index, const float *query_points,
                                        const float *query_lbs, const float *cano2live, int32_t num_exposures, const float *exposure,
                                        const int32_t *pose_idx, const float *d_means3D, const float *d_scales3, const float *d_colors,
                                        float *d_dec_out, float *d_cano2live, float *d_exposure, void *workspace, size_t workspace_bytes,
                                        void *stream_)
{
    GA_REQUIRE(N >= 0 && B >= 1 && B <= kMaxFrames && num_pixels >= N, "bad LBS dims N=%d B=%d pixels=%d", N, B, num_pixels);
    GA_REQUIRE(num_joints == 24 || num_joints == 55, "num_joints %d: 24 (SMPL) or 55 (SMPL-X)", num_joints);
    GA_REQUIRE(lbs_ld % 4 == 0 && lbs_ld >= num_joints, "lbs_ld %d: a multiple of 4 and >= num_joints %d", lbs_ld, num_joints);
    GA_REQUIRE(built_layout(num_joints, lbs_ld), "lbs_ld %d for %d joints is not built (24 joints: 24; 55 joints: 56)", lbs_ld, num_joints);
    GA_REQUIRE(num_exposures >= 1, "num_exposures %d: the exposure table needs at least one row", num_exposures);
    GA_REQUIRE(d_dec_out && d_cano2live && d_exposure, "NULL pointer argument");
    const size_t need = ga_lbs_exposure_workspace_bytes(N, num_joints);
    GA_REQUIRE(workspace_bytes >= need && (workspace || need == 0), "exposure workspace of %zu bytes (need %zu)", workspace_bytes, need);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    GA_CHECK_CUDA(cudaMemsetAsync(d_dec_out, 0, sizeof(float) * 8 * (size_t)num_pixels, stream));
    GA_CHECK_CUDA(cudaMemsetAsync(d_cano2live, 0, sizeof(float) * num_joints * 12 * (size_t)B, stream));
    if (N == 0) {
        GA_CHECK_CUDA(cudaMemsetAsync(d_exposure, 0, sizeof(float) * 12 * (size_t)num_exposures, stream));
        return GA_OK;
    }
    GA_REQUIRE(dec_out && valid_index && query_points && query_lbs && cano2live && exposure && pose_idx && d_means3D && d_scales3 && d_colors,
               "NULL pointer argument");
    ExposureArgs ex;
    ex.F = num_exposures; ex.table = exposure; ex.pidx = pose_idx; ex.partials = static_cast<float *>(workspace);
    const int rc = num_joints == 24
        ? lbs_backward<24, 24, true>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, d_means3D,
                                     d_scales3, d_colors, d_dec_out, d_cano2live, stream, "lbs_kernel<bwd,exposure>", ex)
        : lbs_backward<55, 56, true>(N, B, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, d_means3D,
                                     d_scales3, d_colors, d_dec_out, d_cano2live, stream, "lbs_kernel<bwd,55,exposure>", ex);
    if (rc != GA_OK) return rc;
    const int elems = 12 * num_exposures;
    { ProfScope _ps("lbs_exposure_reduce", stream); lbs_exposure_reduce_kernel<<<cdiv(elems, kReduceWarps), 32 * kReduceWarps, 0, stream>>>(
        num_exposures, B, exposure_ctas(N, num_joints), pose_idx, ex.partials, d_exposure); }
    GA_CHECK_LAUNCH("lbs_exposure_reduce");
    return GA_OK;
}

extern "C" int ga_lbs_forward(int32_t N, int32_t B, float scale_mul, int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index,
                              const float *query_points, const float *query_lbs, const float *cano2live, float *means3D,
                              float *scales3, float *colors, void *stream_)
{
    return ga_lbs_forward_ex(N, B, 24, 24, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live, means3D, scales3,
                             colors, stream_);
}

extern "C" int ga_lbs_backward(int32_t N, int32_t B, int32_t num_pixels, float scale_mul, int64_t dec_frame_stride, const float *dec_out,
                               const int32_t *valid_index, const float *query_points, const float *query_lbs,
                               const float *cano2live, const float *d_means3D, const float *d_scales3, const float *d_colors,
                               float *d_dec_out, float *d_cano2live, void *stream_)
{
    return ga_lbs_backward_ex(N, B, 24, 24, num_pixels, scale_mul, dec_frame_stride, dec_out, valid_index, query_points, query_lbs, cano2live,
                              d_means3D, d_scales3, d_colors, d_dec_out, d_cano2live, stream_);
}
