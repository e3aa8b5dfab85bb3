// Strict-FP32 tiled GEMM skeleton with pluggable operand loaders and epilogues (CUDA-core path).
//
// C[Mg x Ng] (+)= A'[Mg x Kg] * B'[Kg x Ng].  A' and B' are *virtual* matrices produced on the fly by loader functors
// (BatchNorm + Softplus applied while loading, BatchNorm-backward applied while loading, im2col, concatenation, ...)
// so that no activation tensor is ever re-written just to change its form.  The epilogue functor consumes the
// accumulator tile (bias + per-channel statistics, activation backward, split-K atomics, ...).
//
// This is the reference-accuracy path of the decoder MLP / geometry convs (every product is an FP32 FMA); the
// TF32 tensor-core path (mlp_tc.cu) shares the same loaders' semantics and is checked against this one.
#pragma once
#include "common.cuh"

namespace ga {

constexpr int kBK = 16;
constexpr int kGemmThreads = 256;

__device__ __forceinline__ float softplus_f(float z) { return z > 20.f ? z : log1pf(expf(z)); }
__device__ __forceinline__ float sigmoid_f(float z) { return 1.f / (1.f + expf(-z)); }
// fast forms for the TF32 tensor-core path (inputs are rounded to 10 mantissa bits right after): 2 MUFU ops each
__device__ __forceinline__ float softplus_fast(float z) { return fmaxf(z, 0.f) + __logf(1.f + __expf(-fabsf(z))); }
// sigmoid of z = zl / log2(e) given zl: 1 / (1 + 2^-zl) -> MUFU.EX2, FADD, MUFU.RCP
__device__ __forceinline__ float sigmoid_log2(float zl)
{
    float t;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(-zl));
    return __fdividef(1.f, 1.f + t);
}
// softplus of z = zl / log2(e) given zl (the BatchNorm coefficients are pre-multiplied by log2(e) once per kernel):
// ln2 * (max(zl, 0) + log2(1 + 2^-|zl|)) -> FMNMX, MUFU.EX2, FADD, MUFU.LG2, FADD, FMUL
__device__ __forceinline__ float softplus_log2(float zl)
{
    float t, l;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(-fabsf(zl)));
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.f + t));
    return 0.69314718056f * (fmaxf(zl, 0.f) + l);
}
__device__ __forceinline__ float sigmoid_fast(float z) { return __fdividef(1.f, 1.f + __expf(-z)); }

// ---------------------------------------------------------------------------------------------------------------
// Fragment = what one thread holds of a (rows x 16) or (16 x cols) operand tile between global fetch and smem store.
// "K-contiguous" sources (k fastest in memory) are transposed on the way into shared memory; "direct" sources
// (the tile's M or N index fastest in memory) are copied as float4.
// Shared layout: As[k][BM + kPad], Bs[k][BN + kPad].
// ---------------------------------------------------------------------------------------------------------------
constexpr int kPad = 4;

template <int ROWS>
struct FragK {                      // ROWS x 16 tile, k-contiguous source: thread -> rows (tid/4 + 64 i), k quad (tid%4)*4
    static constexpr int kN = ROWS / 64;
    float4 v[kN];
};
template <int ROWS>
__device__ __forceinline__ void store_fragK(float *S, const FragK<ROWS> &f, int tid)
{
    const int kq = (tid & 3) * 4;
#pragma unroll
    for (int i = 0; i < FragK<ROWS>::kN; ++i) {
        const int row = (tid >> 2) + 64 * i;
        S[(kq + 0) * (ROWS + kPad) + row] = f.v[i].x;
        S[(kq + 1) * (ROWS + kPad) + row] = f.v[i].y;
        S[(kq + 2) * (ROWS + kPad) + row] = f.v[i].z;
        S[(kq + 3) * (ROWS + kPad) + row] = f.v[i].w;
    }
}
template <int COLS>
struct FragD {                      // 16 x COLS tile, direct source: thread -> k (tid / (COLS/4) + step i), col quad
    static constexpr int kPerRow = COLS / 4;
    static constexpr int kRowsPerPass = kGemmThreads / kPerRow;
    static constexpr int kN = kBK / kRowsPerPass;
    float4 v[kN];
};
template <int COLS>
__device__ __forceinline__ void store_fragD(float *S, const FragD<COLS> &f, int tid)
{
    const int cq = (tid % FragD<COLS>::kPerRow) * 4;
#pragma unroll
    for (int i = 0; i < FragD<COLS>::kN; ++i) {
        const int k = tid / FragD<COLS>::kPerRow + FragD<COLS>::kRowsPerPass * i;
        *reinterpret_cast<float4 *>(&S[k * (COLS + kPad) + cq]) = f.v[i];
    }
}

// per-channel affine (BatchNorm folded: z = y * a[c] + b[c]) + softplus
struct ChanAffine {
    const float *a, *b;     // nullptr a => raw (no BN / activation)
};

// ---- A loaders (tile = BM rows of Mg x 16 of Kg) ---------------------------------------------------------------

// [raw src0 (K0 cols) | softplus(bn(src1)) (K - K0 cols)], both row-major k-contiguous.  K0 % 4 == 0.
template <int BM>
struct ALoadConcatActK {
    using Frag = FragK<BM>;
    const float *src0; int ld0; int K0;
    const float *src1; int ld1; ChanAffine aff;
    int M, K;
    __device__ __forceinline__ void fetch(Frag &f, int m0, int k0, int tid) const
    {
        const int k = k0 + (tid & 3) * 4;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int m = m0 + (tid >> 2) + 64 * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < M && k < K) {
                if (k < K0) v = *reinterpret_cast<const float4 *>(src0 + (size_t)m * ld0 + k);
                else {
                    const int c = k - K0;
                    v = *reinterpret_cast<const float4 *>(src1 + (size_t)m * ld1 + c);
                    if (aff.a) {
                        const float4 a = *reinterpret_cast<const float4 *>(aff.a + c), b = *reinterpret_cast<const float4 *>(aff.b + c);
                        v.x = softplus_f(fmaf(v.x, a.x, b.x)); v.y = softplus_f(fmaf(v.y, a.y, b.y));
                        v.z = softplus_f(fmaf(v.z, a.z, b.z)); v.w = softplus_f(fmaf(v.w, a.w, b.w));
                    }
                }
            }
            f.v[i] = v;
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragK<BM>(S, f, tid); }
};

// BatchNorm backward applied on load: dY = ga[c] * (dZ - m1[c] - xhat * m2[c]), xhat = (Y - mu[c]) * rstd[c].
// ga == nullptr => dY = dZ (layer without BN).
struct BnBwdCoef {
    const float *ga, *m1, *m2, *mu, *rstd;
};
__device__ __forceinline__ float4 bn_bwd4(const BnBwdCoef &c, int ch, float4 dz, float4 y)
{
    const float4 ga = *reinterpret_cast<const float4 *>(c.ga + ch), m1 = *reinterpret_cast<const float4 *>(c.m1 + ch),
                 m2 = *reinterpret_cast<const float4 *>(c.m2 + ch), mu = *reinterpret_cast<const float4 *>(c.mu + ch),
                 rs = *reinterpret_cast<const float4 *>(c.rstd + ch);
    float4 o;
    o.x = ga.x * (dz.x - m1.x - (y.x - mu.x) * rs.x * m2.x);
    o.y = ga.y * (dz.y - m1.y - (y.y - mu.y) * rs.y * m2.y);
    o.z = ga.z * (dz.z - m1.z - (y.z - mu.z) * rs.z * m2.z);
    o.w = ga.w * (dz.w - m1.w - (y.w - mu.w) * rs.w * m2.w);
    return o;
}

// A'(m, k) = dY[m, k] (k = output channel of the layer), k-contiguous.  For dgrad.
template <int BM>
struct ALoadBnBwdK {
    using Frag = FragK<BM>;
    const float *dZ, *Y; int ld; BnBwdCoef coef; int M, K;
    __device__ __forceinline__ void fetch(Frag &f, int m0, int k0, int tid) const
    {
        const int k = k0 + (tid & 3) * 4;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int m = m0 + (tid >> 2) + 64 * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < M && k < K) {
                v = *reinterpret_cast<const float4 *>(dZ + (size_t)m * ld + k);
                if (coef.ga) v = bn_bwd4(coef, k, v, *reinterpret_cast<const float4 *>(Y + (size_t)m * ld + k));
            }
            f.v[i] = v;
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragK<BM>(S, f, tid); }
};

// A'(mg = out channel, kg = pixel) = dY[pixel, channel]: direct (channel fastest).  For wgrad.
template <int BM>
struct ALoadBnBwdD {
    using Frag = FragD<BM>;
    const float *dZ, *Y; int ld; BnBwdCoef coef; int Mg /*channels*/, Kg /*pixels*/;
    __device__ __forceinline__ void fetch(Frag &f, int m0, int k0, int tid) const
    {
        const int c = m0 + (tid % Frag::kPerRow) * 4;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int p = k0 + tid / Frag::kPerRow + Frag::kRowsPerPass * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < Kg && c < Mg) {
                v = *reinterpret_cast<const float4 *>(dZ + (size_t)p * ld + c);
                if (coef.ga) v = bn_bwd4(coef, c, v, *reinterpret_cast<const float4 *>(Y + (size_t)p * ld + c));
            }
            f.v[i] = v;
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragD<BM>(S, f, tid); }
};

// ---- B loaders (tile = 16 of Kg x BN cols of Ng) ---------------------------------------------------------------

// B'(k, n) = W[n, k], W row-major [Ng, ld] (k-contiguous): transposing.  Forward weights.
template <int BN>
struct BLoadWT {
    using Frag = FragK<BN>;
    const float *W; int ld; int N, K;
    __device__ __forceinline__ void fetch(Frag &f, int n0, int k0, int tid) const
    {
        const int k = k0 + (tid & 3) * 4;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int n = n0 + (tid >> 2) + 64 * i;
            f.v[i] = (n < N && k < K) ? *reinterpret_cast<const float4 *>(W + (size_t)n * ld + k) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragK<BN>(S, f, tid); }
};

// B'(k, n) = Mat[k, n], row-major [Kg, ld] (n-contiguous): direct.  dgrad weights, conv weights.
template <int BN>
struct BLoadDirect {
    using Frag = FragD<BN>;
    const float *Mat; int ld; int N, K;
    __device__ __forceinline__ void fetch(Frag &f, int n0, int k0, int tid) const
    {
        const int n = n0 + (tid % Frag::kPerRow) * 4;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int k = k0 + tid / Frag::kPerRow + Frag::kRowsPerPass * i;
            f.v[i] = (k < K && n < N) ? *reinterpret_cast<const float4 *>(Mat + (size_t)k * ld + n) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragD<BN>(S, f, tid); }
};

// B'(kg = pixel, n = input channel) = [raw src0 | softplus(bn(src1))][pixel, n]: direct.  wgrad activations.
template <int BN>
struct BLoadConcatActD {
    using Frag = FragD<BN>;
    const float *src0; int ld0; int K0;
    const float *src1; int ld1; ChanAffine aff;
    int N /*channels*/, K /*pixels*/;
    __device__ __forceinline__ void fetch(Frag &f, int n0, int k0, int tid) const
    {
        const int n = n0 + (tid % Frag::kPerRow) * 4;
#pragma unroll
        for (int i = 0; i < Frag::kN; ++i) {
            const int p = k0 + tid / Frag::kPerRow + Frag::kRowsPerPass * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < K && n < N) {
                if (n < K0) v = *reinterpret_cast<const float4 *>(src0 + (size_t)p * ld0 + n);
                else {
                    const int c = n - K0;
                    v = *reinterpret_cast<const float4 *>(src1 + (size_t)p * ld1 + c);
                    if (aff.a) {
                        const float4 a = *reinterpret_cast<const float4 *>(aff.a + c), b = *reinterpret_cast<const float4 *>(aff.b + c);
                        v.x = softplus_f(fmaf(v.x, a.x, b.x)); v.y = softplus_f(fmaf(v.y, a.y, b.y));
                        v.z = softplus_f(fmaf(v.z, a.z, b.z)); v.w = softplus_f(fmaf(v.w, a.w, b.w));
                    }
                }
            }
            f.v[i] = v;
        }
    }
    __device__ __forceinline__ void store(float *S, const Frag &f, int tid) const { store_fragD<BN>(S, f, tid); }
};

// ---------------------------------------------------------------------------------------------------------------
// The kernel.  grid = (Mg tiles, Ng tiles, split-K); 256 threads as 16 x 16; each thread owns (BM/16) x (BN/16)
// outputs arranged as float4 groups: rows {ty*4 + i} and {BM/2 + ty*4 + i}, cols likewise (conflict-free LDS.128).
// Register double buffering: the next k-tile is fetched from global while the current one is multiplied.
// ---------------------------------------------------------------------------------------------------------------
template <int BM, int BN>
struct ThreadTile {
    static constexpr int TM = BM / 16, TN = BN / 16;
    static constexpr int RG = TM / 4, CG = TN / 4;   // float4 groups per thread
    __device__ static __forceinline__ int row(int ty, int i) { return (i / 4) * (BM / RG) + ty * 4 + (i % 4); }
    __device__ static __forceinline__ int col(int tx, int j) { return (j / 4) * (BN / CG) + tx * 4 + (j % 4); }
};

template <int BM, int BN, class ALoad, class BLoad, class Epi>
__global__ void __launch_bounds__(kGemmThreads)
gemm_kernel(const ALoad A, const BLoad B, const Epi epi, int Kg, int k_per_split)
{
    using TT = ThreadTile<BM, BN>;
    constexpr int TM = TT::TM, TN = TT::TN;
    __shared__ __align__(16) float As[kBK * (BM + kPad)];
    __shared__ __align__(16) float Bs[kBK * (BN + kPad)];

    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int kbeg = blockIdx.z * k_per_split, kend = min(Kg, kbeg + k_per_split);

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    typename ALoad::Frag fa;
    typename BLoad::Frag fb;
    if (kbeg < kend) { A.fetch(fa, m0, kbeg, tid); B.fetch(fb, n0, kbeg, tid); }
    for (int k0 = kbeg; k0 < kend; k0 += kBK) {
        __syncthreads();
        A.store(As, fa, tid);
        B.store(Bs, fb, tid);
        __syncthreads();
        if (k0 + kBK < kend) { A.fetch(fa, m0, k0 + kBK, tid); B.fetch(fb, n0, k0 + kBK, tid); }
#pragma unroll
        for (int k = 0; k < kBK; ++k) {
            float a[TM], b[TN];
#pragma unroll
            for (int g = 0; g < TT::RG; ++g) {
                const float4 t = *reinterpret_cast<const float4 *>(&As[k * (BM + kPad) + g * (BM / TT::RG) + ty * 4]);
                a[g * 4] = t.x; a[g * 4 + 1] = t.y; a[g * 4 + 2] = t.z; a[g * 4 + 3] = t.w;
            }
#pragma unroll
            for (int g = 0; g < TT::CG; ++g) {
                const float4 t = *reinterpret_cast<const float4 *>(&Bs[k * (BN + kPad) + g * (BN / TT::CG) + tx * 4]);
                b[g * 4] = t.x; b[g * 4 + 1] = t.y; b[g * 4 + 2] = t.z; b[g * 4 + 3] = t.w;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
    }
    __syncthreads();
    epi.template run<BM, BN>(acc, m0, n0, tx, ty, As /* reusable scratch: kBK*(BM+kPad) floats */);
}

// ---- epilogues -------------------------------------------------------------------------------------------------

// C[m, n] = acc (+ bias[n]); optional accumulate into existing C; optional per-column sums of y and y^2 (double).
struct EpiStoreStats {
    float *C; int ld; int M, N;
    const float *bias;       // nullable
    double *sum, *sumsq;     // nullable (both or none): [N] accumulators
    bool accumulate;
    template <int BM, int BN>
    __device__ __forceinline__ void run(float (&acc)[BM / 16][BN / 16], int m0, int n0, int tx, int ty, float *scratch) const
    {
        using TT = ThreadTile<BM, BN>;
        float *s_sum = scratch, *s_sq = scratch + BN;
        if (sum) {
            for (int i = threadIdx.x; i < 2 * BN; i += kGemmThreads) scratch[i] = 0.f;
            __syncthreads();
        }
#pragma unroll
        for (int j = 0; j < TT::TN; ++j) {
            const int n = n0 + TT::col(tx, j);
            const float bv = (bias && n < N) ? bias[n] : 0.f;
            float cs = 0.f, cq = 0.f;
#pragma unroll
            for (int i = 0; i < TT::TM; ++i) {
                const int m = m0 + TT::row(ty, i);
                if (m < M && n < N) {
                    float y = acc[i][j] + bv;
                    acc[i][j] = y;
                    cs += y; cq += y * y;
                }
            }
            if (sum && n < N) { atomicAdd(&s_sum[TT::col(tx, j)], cs); atomicAdd(&s_sq[TT::col(tx, j)], cq); }
        }
        // vectorised stores: each thread writes float4 groups of columns
#pragma unroll
        for (int i = 0; i < TT::TM; ++i) {
            const int m = m0 + TT::row(ty, i);
            if (m >= M) continue;
#pragma unroll
            for (int g = 0; g < TT::CG; ++g) {
                const int n = n0 + TT::col(tx, g * 4);
                if (n + 3 < N) {
                    float4 *p = reinterpret_cast<float4 *>(C + (size_t)m * ld + n);
                    float4 v = make_float4(acc[i][g * 4], acc[i][g * 4 + 1], acc[i][g * 4 + 2], acc[i][g * 4 + 3]);
                    if (accumulate) { const float4 o = *p; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
                    *p = v;
                } else {
                    for (int q = 0; q < 4; ++q)
                        if (n + q < N) {
                            float *p = C + (size_t)m * ld + n + q;
                            *p = accumulate ? (*p + acc[i][g * 4 + q]) : acc[i][g * 4 + q];
                        }
                }
            }
        }
        if (sum) {
            __syncthreads();
            for (int i = threadIdx.x; i < BN; i += kGemmThreads) {
                if (n0 + i < N) { atomicAdd(&sum[n0 + i], (double)s_sum[i]); atomicAdd(&sumsq[n0 + i], (double)s_sq[i]); }
            }
        }
    }
};

// dgrad epilogue.  Columns n < K0: raw gradient w.r.t. the concatenated raw input (store or accumulate into G0).
// Columns n >= K0 (channel c = n - K0 of the previous BN layer): dZ = dX * sigmoid(z), z = y a[c] + b[c];
// store dZ; accumulate per-channel sum(dZ) and sum(dZ * xhat) in double.
struct EpiDgradAct {
    int M, N, K0;
    float *G0; int ld0; bool accumulate0;
    float *dZ; const float *Yprev; int ld1;
    const float *a, *b, *mu, *rstd;      // BN of the previous layer (per channel)
    double *s1, *s2;                     // [N - K0] accumulators: sum dZ, sum dZ*xhat
    template <int BM, int BN>
    __device__ __forceinline__ void run(float (&acc)[BM / 16][BN / 16], int m0, int n0, int tx, int ty, float *scratch) const
    {
        using TT = ThreadTile<BM, BN>;
        float *s_1 = scratch, *s_2 = scratch + BN;
        for (int i = threadIdx.x; i < 2 * BN; i += kGemmThreads) scratch[i] = 0.f;
        __syncthreads();
#pragma unroll
        for (int g = 0; g < TT::CG; ++g) {
            const int n = n0 + TT::col(tx, g * 4);
            if (n >= N) continue;
            if (n < K0) {
#pragma unroll
                for (int i = 0; i < TT::TM; ++i) {
                    const int m = m0 + TT::row(ty, i);
                    if (m >= M) continue;
                    float4 *p = reinterpret_cast<float4 *>(G0 + (size_t)m * ld0 + n);
                    float4 v = make_float4(acc[i][g * 4], acc[i][g * 4 + 1], acc[i][g * 4 + 2], acc[i][g * 4 + 3]);
                    if (accumulate0) { const float4 o = *p; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
                    *p = v;
                }
            } else {
                const int c = n - K0;
                const float4 av = *reinterpret_cast<const float4 *>(a + c), bv = *reinterpret_cast<const float4 *>(b + c),
                             muv = *reinterpret_cast<const float4 *>(mu + c), rsv = *reinterpret_cast<const float4 *>(rstd + c);
                float c1[4] = {0.f, 0.f, 0.f, 0.f}, c2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int i = 0; i < TT::TM; ++i) {
                    const int m = m0 + TT::row(ty, i);
                    if (m >= M) continue;
                    const float4 y = *reinterpret_cast<const float4 *>(Yprev + (size_t)m * ld1 + c);
                    float4 d;
                    d.x = acc[i][g * 4 + 0] * sigmoid_f(fmaf(y.x, av.x, bv.x));
                    d.y = acc[i][g * 4 + 1] * sigmoid_f(fmaf(y.y, av.y, bv.y));
                    d.z = acc[i][g * 4 + 2] * sigmoid_f(fmaf(y.z, av.z, bv.z));
                    d.w = acc[i][g * 4 + 3] * sigmoid_f(fmaf(y.w, av.w, bv.w));
                    *reinterpret_cast<float4 *>(dZ + (size_t)m * ld1 + c) = d;
                    c1[0] += d.x; c1[1] += d.y; c1[2] += d.z; c1[3] += d.w;
                    c2[0] += d.x * (y.x - muv.x) * rsv.x; c2[1] += d.y * (y.y - muv.y) * rsv.y;
                    c2[2] += d.z * (y.z - muv.z) * rsv.z; c2[3] += d.w * (y.w - muv.w) * rsv.w;
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) { atomicAdd(&s_1[TT::col(tx, g * 4 + q)], c1[q]); atomicAdd(&s_2[TT::col(tx, g * 4 + q)], c2[q]); }
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < BN; i += kGemmThreads) {
            const int n = n0 + i;
            if (n < N && n >= K0) { atomicAdd(&s1[n - K0], (double)s_1[i]); atomicAdd(&s2[n - K0], (double)s_2[i]); }
        }
    }
};

// split-K partial product: atomically add the tile into C (fp32).
struct EpiAtomicAdd {
    float *C; int ld; int M, N;
    template <int BM, int BN>
    __device__ __forceinline__ void run(float (&acc)[BM / 16][BN / 16], int m0, int n0, int tx, int ty, float *) const
    {
        using TT = ThreadTile<BM, BN>;
#pragma unroll
        for (int i = 0; i < TT::TM; ++i) {
            const int m = m0 + TT::row(ty, i);
            if (m >= M) continue;
#pragma unroll
            for (int j = 0; j < TT::TN; ++j) {
                const int n = n0 + TT::col(tx, j);
                if (n < N) atomicAdd(C + (size_t)m * ld + n, acc[i][j]);
            }
        }
    }
};

}  // namespace ga
