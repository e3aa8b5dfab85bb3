// Decoder-MLP layers on the tensor cores (wgmma.mma_async TF32, fp32 accumulators in registers), warp-specialised.
//
// Forward: one persistent CTA per SM computes  Y[M,128] (+)= act(bn(X))[M,K] * W[128,K]^T + bias  for its share of 64-pixel tiles,
// as the TRANSPOSED product  Y^T[out, px] = W[out, K] * act(bn(X))[px, K]^T, with three warpgroups:
//   producer  (warpgroup 0): the raw (pre-BatchNorm) input rows travel global -> shared with 16-byte cp.async, each piece straight to
//              its place in the 128-byte-swizzled K-major tile image, up to four tiles ahead over six 32 KB stages; the thread that
//              copied a piece converts it IN PLACE (BatchNorm + Softplus in the log2 domain, TF32 rounding) once it has landed and
//              hands the stage to the consumers through the stage's `full` mbarrier
//   consumers (warpgroups 1, 2): warpgroup c owns output channels 64 c .. 64 c + 63; its slice of W lives in registers as wgmma A
//              fragments for the whole launch (zero past K), the tile image is the B operand (16 wgmma m64n64k8 per tile, a uniform
//              sequence the compiler does not have to fence one by one; channels past K are zero-filled); the stage goes back to
//              the producer through its `empty` mbarrier as soon as the MMAs have retired, then the epilogue works from the
//              accumulators: bias, the fan-in's existing Y, the layer's BatchNorm sum / sum-of-squares (per channel, reduced over the
//              four lanes that share a channel); the values go to the warpgroup's own 16 KB staging half (its two 32-channel chunks,
//              laid out like the X image, which is the TMA SWIZZLE_128B box) and one thread stores the half with two TMA tensor
//              stores, which drain while the warpgroup runs the next tile's MMAs (the half is rewritten once the stores have read it)
// setmaxnreg moves registers from the producer (a few per element in flight) to the consumers (W fragments + accumulators).
//
// TF32 is what the reference computes these 1x1 convolutions in on any Ampere+ GPU (cuDNN allow_tf32 default,
// SURVEY.md §8 a-4); the strict-FP32 CUDA-core path (gemm.cuh) remains selectable and is the GPU-side reference.
#include <cudaTypedefs.h>

#include "gemm.cuh"
#include "tc_common.cuh"

namespace ga {
namespace {

using namespace tc;

constexpr size_t kMaxSmemPerBlock = 232448;          // sm_90 opt-in limit of dynamic shared memory per block (227 KB)

// Tensor map of the fp32 matrix [rows][cols] (leading dimension ld floats) in 128-byte-swizzled boxes of 32 columns x box_rows rows,
// the K-major image layout of tc_common.cuh.  cuTensorMapEncodeTiled is a driver function; it is reached through the runtime's
// entry-point query so that the library links the runtime only.
int make_tmap(CUtensorMap *m, const float *base, int cols, int rows, int ld, int box_rows)
{
    static PFN_cuTensorMapEncodeTiled_v12000 encode = [] {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            fn = nullptr;
        return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    }();
    GA_REQUIRE(encode, "cuTensorMapEncodeTiled is not available from the driver");
    GA_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor-core layer: the output must be 16-byte aligned");
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)ld * sizeof(float)};
    const cuuint32_t box[2] = {32, (cuuint32_t)box_rows}, estr[2] = {1, 1};
    const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    GA_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): cols %d rows %d ld %d", (int)r, cols, rows, ld);
    return GA_OK;
}

constexpr int kTcThreads = 3 * 128;                  // producer warpgroup + two consumer warpgroups
constexpr int kProdRegs = 80, kConsRegs = 208;       // setmaxnreg split: 128 x 80 + 256 x 208 <= 384 x 168 (the launch allocation)
static_assert(128 * kProdRegs + 256 * kConsRegs <= kTcThreads * 168, "the consumers' registers must come from the producer's");

constexpr int kTPx = 64, kTStages = 6;
constexpr int kTLook = 4;                            // tiles of copies in flight (a stage is refilled two tiles after it was read)
constexpr int kTChunk = kTPx * 128;                  // 8 KB: [64 px rows][32 channels]
constexpr int kTStageBytes = 4 * kTChunk;            // 32 KB: K <= 128
static_assert(kTLook <= kTStages - 2, "lookahead must leave the stages being converted and read alone");

struct TcFwdParams {
    CUtensorMap ymap;              // Y [M][128] (leading dimension ldy) in boxes of 32 channels x 64 pixels
    const float *X; int ldx; int K;
    const float *a, *b;            // folded BatchNorm of the producer layer (nullptr: raw input, no activation)
    const float *W; int ldw;       // [128][K] row-major
    const float *bias;             // nullable
    int accumulate;
    double *sum, *sumsq;           // nullable
    int M;
};

struct alignas(1024) TcFwdSmem {
    unsigned char x[kTStages][kTStageBytes];         // X tile: [4 chunks][64 px rows][128 B], K-major, 128-byte swizzle
    unsigned char ys[2][2 * kTChunk];                // Y staging of consumer warpgroup c: its 2 chunks of 32 channels, the X tile's layout
    float sa[128], sb[128];
    uint64_t full[kTStages], empty[kTStages];        // producer -> consumers (128 arrivals), consumers -> producer (256 arrivals)
    uint64_t yload[2];                               // accumulate: the existing Y of the tile has landed in ys[c] (TMA load)
};
static_assert(sizeof(TcFwdSmem) + 1024 <= kMaxSmemPerBlock, "forward shared memory");

__global__ void __launch_bounds__(kTcThreads, 1)
tc_fwd_kernel(const __grid_constant__ TcFwdParams p)
{
    extern __shared__ unsigned char smem_raw[];
    TcFwdSmem &sm = *reinterpret_cast<TcFwdSmem *>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int num_tiles = (p.M + kTPx - 1) / kTPx;
    const int gstep = gridDim.x;
    const int ntl = (num_tiles - (int)blockIdx.x + gstep - 1) / gstep;       // tiles of this CTA (grid <= tiles: >= 1)
    const int M = p.M;
    if (tid < kTStages) { mbar_init(smem_u32(&sm.full[tid]), 128); mbar_init(smem_u32(&sm.empty[tid]), 256); }
    if (tid < 2) { mbar_init(smem_u32(&sm.yload[tid]), 1); fence_proxy_async(); }   // completed by TMA loads (async proxy)
    for (int i = tid; i < p.K; i += kTcThreads) { sm.sa[i] = p.a ? p.a[i] : 1.f; sm.sb[i] = p.a ? p.b[i] : 0.f; }
    __syncthreads();
    const uint32_t x0s = smem_u32(sm.x[0]);

    if (warp < 4) {
        // ---- producer: warp w owns channel chunk c = w and pixel rows r0 + 8 i (i = 0..7) for r0 = 4 h + lane / 8, h = 0, 1; a warp
        // instruction covers 4 rows x 128 B
        setmaxnreg_dec<kProdRegs>();
        const int rl = lane >> 3, u = lane & 7;
        const int c = warp;
        const int k = c * 32 + u * 4;
        const bool kin = k < p.K;
        float4 av = make_float4(1.f, 1.f, 1.f, 1.f), bv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kin) { av = *reinterpret_cast<const float4 *>(&sm.sa[k]); bv = *reinterpret_cast<const float4 *>(&sm.sb[k]); }
        const bool act = p.a != nullptr;
        {   // log2 domain: z * log2(e) comes straight out of the FMA
            const float L2E = 1.44269504089f;
            av.x *= L2E; av.y *= L2E; av.z *= L2E; av.w *= L2E; bv.x *= L2E; bv.y *= L2E; bv.z *= L2E; bv.w *= L2E;
        }
        const int ldx = p.ldx;
        uint32_t soffs[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r0 = 4 * h + rl;
            const uint32_t soff = (uint32_t)c * kTChunk + sw128_offset(r0, u);   // + i * 1024
            soffs[h] = soff;
        }
        const float *x0 = p.X + (size_t)rl * ldx + k;
        auto issue = [&](int j) {
            const int st = j % kTStages;
            // every producer thread waits (also those without copies): none may arrive on a stage's `full` barrier a round early
            if (j < ntl && j >= kTStages) mbar_wait(smem_u32(&sm.empty[st]), ((j / kTStages) & 1) ^ 1);   // tile j - kTStages is read
            if (j < ntl) {
                const int t = blockIdx.x + j * gstep;
                const uint32_t dst = x0s + (uint32_t)st * kTStageBytes;
                const float *src = x0 + (size_t)t * kTPx * ldx;
                const bool whole = (t + 1) * kTPx <= M;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int r = 4 * h + rl + 8 * i;
                        const bool ok = kin && (whole || t * kTPx + r < M);      // rows >= M and channels >= K are zero-filled
                        cp_async16(dst + soffs[h] + i * 1024, ok ? src + (size_t)(4 * h + 8 * i) * ldx : p.X, ok);
                    }
            }
            cp_async_commit();                             // one group per tile (empty past the end): the wait count stays uniform
        };
        for (int j = 0; j < kTLook; ++j) issue(j);
        for (int j = 0; j < ntl; ++j) {
            const int st = j % kTStages;
            cp_async_wait<kTLook - 1>();
            if (kin) {                                     // channels >= K stay zero: the MMAs multiply them by zero weights
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    unsigned char *xs = sm.x[st] + soffs[h];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        float4 x = *reinterpret_cast<const float4 *>(xs + i * 1024);
                        if (act) {
                            x.x = softplus_log2(fmaf(x.x, av.x, bv.x)); x.y = softplus_log2(fmaf(x.y, av.y, bv.y));
                            x.z = softplus_log2(fmaf(x.z, av.z, bv.z)); x.w = softplus_log2(fmaf(x.w, av.w, bv.w));
                        }
                        *reinterpret_cast<float4 *>(xs + i * 1024) = to_tf32(x);   // rows >= M hold act(bn(0)): their columns are never stored
                    }
                }
            }
            fence_proxy_async();                           // the converted pieces are read by the tensor cores (async proxy)
            mbar_arrive(smem_u32(&sm.full[st]));
            issue(j + kTLook);
        }
        cp_async_wait<0>();
        return;
    }

    // ---- consumers
    setmaxnreg_inc<kConsRegs>();
    const int g = lane >> 2, t4 = lane & 3;
    // W slice of this warp as A fragments: rows (output channels) oc, oc + 8; K columns 8 ks + t4, + 4 (zero past K)
    const int oc = 16 * (warp - 4) + g;                                      // warpgroup c = (warp - 4) / 4: channels 64 c .. 64 c + 63
    uint32_t wa[16][4];
#pragma unroll
    for (int ks = 0; ks < 16; ++ks) {
        const int k = 8 * ks + t4;
        const bool ok = 8 * ks < p.K;
        wa[ks][0] = __float_as_uint(ok ? to_tf32(p.W[(size_t)oc * p.ldw + k]) : 0.f);
        wa[ks][1] = __float_as_uint(ok ? to_tf32(p.W[(size_t)(oc + 8) * p.ldw + k]) : 0.f);
        wa[ks][2] = __float_as_uint(ok ? to_tf32(p.W[(size_t)oc * p.ldw + k + 4]) : 0.f);
        wa[ks][3] = __float_as_uint(ok ? to_tf32(p.W[(size_t)(oc + 8) * p.ldw + k + 4]) : 0.f);
    }
    const float bias0 = p.bias ? p.bias[oc] : 0.f, bias1 = p.bias ? p.bias[oc + 8] : 0.f;
    // staging: this warpgroup's channels 64 c .. 64 c + 63 are columns ocl = oc - 64 c of its half; thread 0 of the warpgroup moves it
    const int wg = (warp - 4) >> 2, ocl = oc - 64 * wg;
    const bool leader = (tid & 127) == 0;
    unsigned char *ys = sm.ys[wg];
    const uint32_t ys_u = smem_u32(ys), yload = smem_u32(&sm.yload[wg]);
    double dsum[2] = {0.0, 0.0}, dsq[2] = {0.0, 0.0};
    for (int j = 0; j < ntl; ++j) {
        const int tile = blockIdx.x + j * gstep, st = j % kTStages;
        const uint32_t xs_u = x0s + (uint32_t)st * kTStageBytes;
        if (leader) {
            bulk_wait_read<0>();                       // the stores of tile j - 1 have read the staging half
            if (p.accumulate) {                        // the existing Y lands in the half while the MMAs run
                mbar_arrive_expect_tx(yload, 2 * kTChunk);
#pragma unroll
                for (int c = 0; c < 2; ++c) tma_load_2d(ys_u + c * kTChunk, &p.ymap, yload, 64 * wg + 32 * c, tile * kTPx);
            }
        }
        mbar_wait(smem_u32(&sm.full[st]), (j / kTStages) & 1);

        float acc[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 16; ++ks) wgmma_tf32_n64(acc, wa[ks], wgmma_desc(kstep_addr(xs_u, ks, kTChunk)));
        wgmma_commit();
        warpgroup_bar(2 + wg);                         // the staging half is free (under the MMAs)
        wgmma_wait<0>();
        wgmma_fence_operand(acc);
        mbar_arrive(smem_u32(&sm.empty[st]));
        if (p.accumulate) mbar_wait(yload, j & 1);

        // ---- epilogue: acc[nt] = {Y^T(oc, px), Y^T(oc, px + 1), Y^T(oc + 8, px), Y^T(oc + 8, px + 1)}, px = 8 nt + 2 t4
        float cs[2] = {0.f, 0.f}, cq[2] = {0.f, 0.f};
        const int rows = M - tile * kTPx;              // valid pixels of this tile; the stores clip the rest
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int px = 8 * nt + 2 * t4 + e;
                float *y0 = reinterpret_cast<float *>(ys + kmajor_off(px, ocl, kTChunk));
                float *y1 = reinterpret_cast<float *>(ys + kmajor_off(px, ocl + 8, kTChunk));
                float v0 = acc[nt][e] + bias0, v1 = acc[nt][2 + e] + bias1;
                if (p.accumulate) { v0 += *y0; v1 += *y1; }
                *y0 = v0; *y1 = v1;
                if (px < rows) {
                    cs[0] += v0; cq[0] = fmaf(v0, v0, cq[0]);
                    cs[1] += v1; cq[1] = fmaf(v1, v1, cq[1]);
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) { dsum[h] += (double)cs[h]; dsq[h] += (double)cq[h]; }
        fence_proxy_async();                           // the staged values are read by the TMA stores (async proxy)
        warpgroup_bar(2 + wg);
        if (leader) {
#pragma unroll
            for (int c = 0; c < 2; ++c) tma_store_2d(&p.ymap, ys_u + c * kTChunk, 64 * wg + 32 * c, tile * kTPx);
            bulk_commit();
        }
    }
    if (leader) bulk_wait<0>();                        // nothing in flight when the CTA exits
    if (p.sum) {                                       // the four lanes of a channel meet by shuffles: 2 atomics per channel per CTA
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) {
                dsum[h] += __shfl_xor_sync(0xffffffffu, dsum[h], o);
                dsq[h] += __shfl_xor_sync(0xffffffffu, dsq[h], o);
            }
            if (t4 == 0) { atomicAdd(&p.sum[oc + 8 * h], dsum[h]); atomicAdd(&p.sumsq[oc + 8 * h], dsq[h]); }
        }
    }
}

}  // namespace

// Host-side launcher shared by the decoder orchestration and the unit-test entry point.
int launch_tc_fwd(const float *X, int ldx, int K, const float *a, const float *b, const float *W, int ldw, const float *bias, float *Y,
                  int ldy, int accumulate, double *sum, double *sumsq, int M, cudaStream_t st)
{
    GA_REQUIRE(K % 8 == 0 && K >= 8 && K <= 128, "tensor-core layer: K=%d must be a multiple of 8 in [8,128]", K);
    GA_REQUIRE(ldx % 4 == 0 && ldw % 4 == 0 && ldy % 4 == 0, "tensor-core layer: leading dimensions must be multiples of 4");
    TcFwdParams p{{}, X, ldx, K, a, b, W, ldw, bias, accumulate, sum, sumsq, M};
    if (int rc = make_tmap(&p.ymap, Y, 128, M, ldy, kTPx)) return rc;
    static PerDeviceOnce attr_t_set;
    if (attr_t_set.first()) {
        GA_CHECK_CUDA(cudaFuncSetAttribute(tc_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcFwdSmem) + 1024));
    }
    const int tiles = cdiv(M, kTPx), sms = num_sms();
    const int grid = tiles < sms ? tiles : sms;
    {
        ProfScope _ps("mlp_tc_fwd", st);
        tc_fwd_kernel<<<grid, kTcThreads, sizeof(TcFwdSmem) + 1024, st>>>(p);
    }
    GA_CHECK_LAUNCH("tc_fwd_kernel");
    return GA_OK;
}

}  // namespace ga

// Unit-test / building-block entry: Y[M,128] (+)= act(bn(X))[M,K] W[128,K]^T + bias on the tensor cores.
extern "C" int ga_tc_linear_forward(int32_t M, int32_t K, const float *X, int32_t ldx, const float *bn_a, const float *bn_b, const float *W,
                                    int32_t ldw, const float *bias, float *Y, int32_t ldy, int32_t accumulate, double *sum, double *sumsq,
                                    void *stream)
{
    GA_REQUIRE(M > 0 && X && W && Y, "bad arguments");
    return ga::launch_tc_fwd(X, ldx, K, bn_a, bn_b, W, ldw, bias, Y, ldy, accumulate, sum, sumsq, M, static_cast<cudaStream_t>(stream));
}

// =====================================================================================================================
// Backward of one hidden layer on the tensor cores: data gradient AND weight gradient from ONE pass over the tile.
//
//   G  = dY_l      [px, out] = ga (dZ_l - m1 - xhat_l m2)          BatchNorm backward applied while loading (dZ_l, Y_l)
//   X  = x_l       [px, in ] = softplus(a Y_{l-1} + b)             recomputed while loading Y_{l-1}
//   dX^T [in, px]  = W_l^T G^T  computed TRANSPOSED: consumer warpgroup c owns input channels 64 c .. 64 c + 63, whose W^T slice lives
//                               in registers as wgmma A fragments for the whole launch; B = the G image (K-major in the output channel)
//   dW_l [out,in] += G^T X      K = pixel: consumer warpgroup c accumulates output rows 64 c .. 64 c + 63 x all 128 input columns in
//                               registers for the whole launch (A = G^T fragments read from the G image, B = the TRANSPOSED X image
//                               [in][px], K-major in the pixel), one flush (8-byte vector reductions) at the end
//   dZ_{l-1} = dX * sigmoid(z_{l-1})   (sigmoid(z_{l-1}) and xhat_{l-1} recovered from x = softplus(z) in the X tile: no re-read)
// Warp-specialised like the forward: the producer warpgroup copies the raw operands global -> shared with 16-byte cp.async (no
// register behind a load in flight), two 32-pixel tiles ahead over four 48 KB stages, converts them (G in place; X, after a
// producer-only barrier, from the landed Y_{l-1} pieces of any producer thread, written transposed over the raw Y_l) and hands each
// stage over through mbarriers; the consumers run the data-gradient MMAs, then the weight-gradient MMAs, whose completion they only wait for after the
// epilogue.  The epilogue stages dZ_{l-1} (or the raw dX) in the warpgroup's own 8 KB half of a staging tile laid out like the G image
// (the TMA SWIZZLE_128B box), and one thread moves it with TMA tensor stores, or tensor reduce-adds for the accumulating mode; a
// mode that finishes on top of the existing values TMA-loads them into the half under the MMAs.
// =====================================================================================================================
namespace ga {
namespace {

constexpr int kPx = 32;
constexpr int kBStages = 4, kLook = 2;    // tiles of raw operand copies in flight (a stage is refilled two tiles after it was read)
constexpr int kGkChunk = kPx * 128;       // 4 KB: [32 px rows][32 channels]
constexpr int kGkTile = 4 * kGkChunk;     // 16 KB
constexpr int kXtTile = 128 * 128;        // 16 KB: transposed X [128 input channels][32 px], K-major in the pixel
static_assert(kXtTile == kGkTile, "X is written over the raw Y_l");
static_assert(kLook <= kBStages - 2, "lookahead must leave the stages being converted and read alone");

struct TcBwdParams {
    CUtensorMap omap;                                  // dZprev [M][kin] (leading dimension ldo) in boxes of 32 channels x 32 pixels
    const float *dZ, *Y; int ldg;                      // layer l: [M][ldg], 128 output channels from the pointer
    const float *ga, *m1, *m2, *mu, *rstd;             // BatchNorm backward of layer l (ga == nullptr: G = dZ)
    const float *Yprev; int ldp;                       // layer l-1 pre-BN output, 128 channels
    const float *pa, *pb, *pmu, *prstd;                // BatchNorm (folded) of layer l-1
    const float *W; int ldw;                           // [128 out][128 in]
    float *dW; int lddw;                               // += (atomics)
    int mode;                                          // 0 final, 1 store raw dX, 2 accumulate raw dX, 3 final on (existing + dX)
    double *s1, *s2;
    int M;
    int kin;                                           // valid input channels (128, or 72 for the [features|uv] input)
    int x_raw;                                         // X = Yprev as is (the network input: no BatchNorm / Softplus; modes 1, 2 only)
};

struct alignas(1024) TcBwdSmem {
    unsigned char gk[kBStages][kGkTile];               // G   rows = pixel, K = output channel (K-major); dZ lands here
    unsigned char yx[kBStages][kXtTile];               // raw Y_l (gk's layout) for the G conversion, then X: rows = input channel, K = pixel
    unsigned char xm[kBStages][kXtTile];               // raw Y_{l-1}, pixel-major: rows = pixel, 32-byte pieces XOR px % 4
    unsigned char os[2][2 * kGkChunk];                 // dZ_{l-1} staging of consumer warpgroup c: its 2 chunks of 32 channels, gk's layout
    float gA[128], gB[128], gC[128];                   // dY = gA dZ + gB Y + gC  (BatchNorm backward folded to two FMAs)
    float pa[128], pb[128], pbeta[128], pinvg[128];    // layer l-1: z log2e = y pa + pb ; xhat = (z - pbeta) * pinvg
    uint64_t full[kBStages], empty[kBStages];          // producer -> consumers (128 arrivals), consumers -> producer (256 arrivals)
    uint64_t oload[2];                                 // mode 3: the existing values of the tile have landed in os[c] (TMA load)
};
static_assert(sizeof(TcBwdSmem) + 1024 <= kMaxSmemPerBlock, "backward shared memory");

__global__ void __launch_bounds__(kTcThreads, 1)
tc_bwd_kernel(const __grid_constant__ TcBwdParams p)
{
    extern __shared__ unsigned char smem_raw[];
    TcBwdSmem &sm = *reinterpret_cast<TcBwdSmem *>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int M = p.M;
    const int num_tiles = (M + kPx - 1) / kPx;
    const int gstep = gridDim.x;
    const int ntl = (num_tiles - (int)blockIdx.x + gstep - 1) / gstep;       // tiles of this CTA (grid <= tiles: >= 1)
    if (tid < kBStages) { mbar_init(smem_u32(&sm.full[tid]), 128); mbar_init(smem_u32(&sm.empty[tid]), 256); }
    if (tid < 2) { mbar_init(smem_u32(&sm.oload[tid]), 1); fence_proxy_async(); }   // completed by TMA loads (async proxy)
    for (int i = tid; i < 128; i += kTcThreads) {
        if (p.ga) {   // ga (dZ - m1 - (Y - mu) rstd m2)
            const float ga = p.ga[i], k = p.rstd[i] * p.m2[i];
            sm.gA[i] = ga; sm.gB[i] = -ga * k; sm.gC[i] = ga * (k * p.mu[i] - p.m1[i]);
        } else { sm.gA[i] = 1.f; sm.gB[i] = 0.f; sm.gC[i] = 0.f; }
        if (p.x_raw) { sm.pa[i] = 1.f; sm.pb[i] = 0.f; sm.pbeta[i] = 0.f; sm.pinvg[i] = 0.f; }
        else {
            // folded BatchNorm of layer l-1 in the log2 domain; xhat = (y - mu) rstd = (z - beta) / gamma with
            // gamma = a / rstd, beta = b + mu a  (a, b: folded scale / shift)
            const float a = p.pa[i], b = p.pb[i];
            sm.pa[i] = a * 1.44269504089f; sm.pb[i] = b * 1.44269504089f;
            sm.pbeta[i] = b + p.pmu[i] * a; sm.pinvg[i] = p.prstd[i] / a;
        }
    }
    __syncthreads();
    const uint32_t gk0 = smem_u32(sm.gk[0]), yx0 = smem_u32(sm.yx[0]), xm0 = smem_u32(sm.xm[0]);

    if (warp < 4) {
        // ---- producer.  Copies: warp w owns the 32-channel chunk jc = w (its BatchNorm coefficients are thread constants) and pixel
        // rows p0 + 8 e for p0 = 4 h + lane / 8, h = 0, 1, of dZ, Y_l and Y_{l-1}; a warp instruction covers 4 pixels x 128 B
        // (full-line global requests).  The pixel-major image of Y_{l-1} (32-byte pieces XOR px % 4):
        //     byte(px, c) = (c / 32) * kGkChunk + px * 128 + ((((c % 32) / 8) ^ (px % 4)) * 32) + (c % 8) * 4
        // keeps a pixel's 32 channels one permuted 128-byte row, like the K-major image (16-byte units XOR px % 8).
        // X conversion: lane owns pixels 4 q .. 4 q + 3 (q = lane / 4) of channel groups cg = 4 (2 w + b) + lane % 4, b = 0, 1
        // (16-byte pieces of 4 channels): a 4 x 4 block per b that it writes transposed as four 16-byte pieces of the X image.
        setmaxnreg_dec<kProdRegs>();
        const int c16 = lane & 7, pxl = lane >> 3, jc = warp;
        const int ch = jc * 32 + c16 * 4;                                    // this thread's 4 channels of G
        uint32_t k_offs[2], mn_offs[2];                                      // + e * 1024
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int p0 = 4 * h + pxl;                                      // p0 % 4 == pxl
            const uint32_t k_off = (uint32_t)jc * kGkChunk + (uint32_t)p0 * 128u + (uint32_t)((c16 ^ p0) << 4);
            const uint32_t mn_off = (uint32_t)jc * kGkChunk + (uint32_t)p0 * 128u + (uint32_t)((((c16 >> 1) ^ pxl) << 5) | ((c16 & 1) << 4));
            k_offs[h] = k_off; mn_offs[h] = mn_off;
        }
        const int q = lane >> 2;
        int cgs[2];
#pragma unroll
        for (int b = 0; b < 2; ++b) cgs[b] = 4 * (2 * warp + b) + (lane & 3);
        const bool has_y = p.ga != nullptr, raw = p.x_raw != 0, okc = ch < p.kin;
        const int ldg = p.ldg, ldp = p.ldp;
        const float *dz0 = p.dZ + (size_t)pxl * ldg + ch, *y0 = (has_y ? p.Y : p.dZ) + (size_t)pxl * ldg + ch;
        const float *x0 = p.Yprev + (size_t)pxl * ldp + ch;
        const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
        auto issue = [&](int jt) {
            if (jt < ntl) {
                const int t = blockIdx.x + jt * gstep, st = jt % kBStages;
                if (jt >= kBStages) mbar_wait(smem_u32(&sm.empty[st]), ((jt / kBStages) & 1) ^ 1);   // tile jt - kBStages is read
                const uint32_t dk = gk0 + (uint32_t)st * kGkTile, dy = yx0 + (uint32_t)st * kXtTile, dx = xm0 + (uint32_t)st * kXtTile;
                const float *pz = dz0 + (size_t)t * kPx * ldg, *py = y0 + (size_t)t * kPx * ldg, *px = x0 + (size_t)t * kPx * ldp;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < kPx / 8; ++e) {
                        const int r = 4 * h + 8 * e;                             // + pxl
                        const bool ok = t * kPx + r + pxl < M;                   // rows >= M are zero-filled
                        cp_async16(dk + k_offs[h] + e * 1024, ok ? pz + (size_t)r * ldg : p.dZ, ok);
                        if (has_y) cp_async16(dy + k_offs[h] + e * 1024, ok ? py + (size_t)r * ldg : p.dZ, ok);
                        cp_async16(dx + mn_offs[h] + e * 1024, ok && okc ? px + (size_t)r * ldp : p.Yprev, ok && okc);   // channels past kin are never read
                    }
            }
            cp_async_commit();                             // one group per tile (empty past the end): the wait count stays uniform
        };
        for (int jt = 0; jt < kLook; ++jt) issue(jt);

        for (int jt = 0; jt < ntl; ++jt) {
            const int st = jt % kBStages;
            const int m0 = (blockIdx.x + jt * gstep) * kPx;
            const bool ragged = m0 + kPx > M;
            cp_async_wait<kLook - 1>();
            {   // G = gA dZ + gB Y + gC -> K-major image, in place over dZ
                const float4 cA = *reinterpret_cast<const float4 *>(&sm.gA[ch]), cB = *reinterpret_cast<const float4 *>(&sm.gB[ch]),
                             cC = *reinterpret_cast<const float4 *>(&sm.gC[ch]);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    unsigned char *gk = sm.gk[st] + k_offs[h], *ym = sm.yx[st] + k_offs[h];
#pragma unroll
                    for (int e = 0; e < kPx / 8; ++e) {
                        const bool row_ok = !ragged || m0 + 4 * h + 8 * e + pxl < M;
                        const float4 za = *reinterpret_cast<const float4 *>(gk + e * 1024);
                        const float4 ya = has_y ? *reinterpret_cast<const float4 *>(ym + e * 1024) : za;
                        float4 o;
                        o.x = fmaf(cA.x, za.x, fmaf(cB.x, ya.x, cC.x)); o.y = fmaf(cA.y, za.y, fmaf(cB.y, ya.y, cC.y));
                        o.z = fmaf(cA.z, za.z, fmaf(cB.z, ya.z, cC.z)); o.w = fmaf(cA.w, za.w, fmaf(cB.w, ya.w, cC.w));
                        if (!row_ok) o = zero4;                               // rows >= M carry zeros (gC alone would not be zero)
                        *reinterpret_cast<float4 *>(gk + e * 1024) = to_tf32(o);
                    }
                }
            }
            // every raw Y_l piece of the tile has been read (X may overwrite them), and every producer thread's Y_{l-1} copies have landed
            warpgroup_bar(1);
            // X = softplus(bn(Y_{l-1})) written transposed: channel c's pixels 4 q .. 4 q + 3 are the 16-byte unit q of row c of the
            // K-major image
#pragma unroll
            for (int b = 0; b < 2; ++b) {
                const int c0 = 4 * cgs[b];
                const float4 av = *reinterpret_cast<const float4 *>(&sm.pa[c0]), bv = *reinterpret_cast<const float4 *>(&sm.pb[c0]);
                const bool okc = c0 < p.kin;
                float4 xv[4];
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    float4 x = *reinterpret_cast<const float4 *>(sm.xm[st] + mnmajor_off(4 * q + r, c0, kGkChunk));
                    if (!raw) {
                        x.x = softplus_log2(fmaf(x.x, av.x, bv.x)); x.y = softplus_log2(fmaf(x.y, av.y, bv.y));
                        x.z = softplus_log2(fmaf(x.z, av.z, bv.z)); x.w = softplus_log2(fmaf(x.w, av.w, bv.w));
                    }
                    if (!okc || (ragged && m0 + 4 * q + r >= M)) x = zero4;   // softplus(bn(0)) is not 0: rows >= M must be
                    xv[r] = to_tf32(x);
                }
                unsigned char *xt = sm.yx[st];
                *reinterpret_cast<float4 *>(xt + sw128_offset(c0 + 0, q)) = make_float4(xv[0].x, xv[1].x, xv[2].x, xv[3].x);
                *reinterpret_cast<float4 *>(xt + sw128_offset(c0 + 1, q)) = make_float4(xv[0].y, xv[1].y, xv[2].y, xv[3].y);
                *reinterpret_cast<float4 *>(xt + sw128_offset(c0 + 2, q)) = make_float4(xv[0].z, xv[1].z, xv[2].z, xv[3].z);
                *reinterpret_cast<float4 *>(xt + sw128_offset(c0 + 3, q)) = make_float4(xv[0].w, xv[1].w, xv[2].w, xv[3].w);
            }
            fence_proxy_async();                           // the converted images are read by the tensor cores (async proxy)
            mbar_arrive(smem_u32(&sm.full[st]));
            issue(jt + kLook);
        }
        cp_async_wait<0>();
        return;
    }

    // ---- consumers
    setmaxnreg_inc<kConsRegs>();
    const int g = lane >> 2, t4 = lane & 3;
    // W^T slice of this warp as A fragments: rows (input channels) ic, ic + 8; K columns (output channels) 8 ks + t4, + 4.  The same
    // index is the output channel of this thread's weight-gradient rows.
    const int ic = 16 * (warp - 4) + g;
    uint32_t wa[16][4];
#pragma unroll
    for (int ks = 0; ks < 16; ++ks) {
        const int o = 8 * ks + t4;
        wa[ks][0] = __float_as_uint(ic < p.kin ? to_tf32(p.W[(size_t)o * p.ldw + ic]) : 0.f);
        wa[ks][1] = __float_as_uint(ic + 8 < p.kin ? to_tf32(p.W[(size_t)o * p.ldw + ic + 8]) : 0.f);
        wa[ks][2] = __float_as_uint(ic < p.kin ? to_tf32(p.W[(size_t)(o + 4) * p.ldw + ic]) : 0.f);
        wa[ks][3] = __float_as_uint(ic + 8 < p.kin ? to_tf32(p.W[(size_t)(o + 4) * p.ldw + ic + 8]) : 0.f);
    }
    // ---- per-thread constants of the epilogue: input channels ic + 8 h
    const bool final_mode = p.mode == 0 || p.mode == 3;
    // staging: this warpgroup's input channels 64 c .. 64 c + 63 are columns icl = ic - 64 c of its half; its chunks at or past kin are
    // never moved.  Thread 0 of the warpgroup moves the half.
    const int wg = (warp - 4) >> 2, icl = ic - 64 * wg;
    const int nchunks = max(0, min(2, (p.kin - 64 * wg + 31) / 32));
    const bool load_existing = p.mode == 3 && nchunks > 0;   // mode 2 adds in L2 (TMA reduce-add): the SM reads nothing
    const bool leader = (tid & 127) == 0;
    unsigned char *os = sm.os[wg];
    const uint32_t os_u = smem_u32(os), oload = smem_u32(&sm.oload[wg]);
    float cinvg[2], cbg[2], cl2g[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        // xhat = (z - beta) / gamma with z = x + ln2 * log2(sigmoid):  xhat = ln2/gamma * ls + (x / gamma - beta / gamma)
        const int c = ic + 8 * h;
        cinvg[h] = sm.pinvg[c]; cbg[h] = sm.pbeta[c] * cinvg[h]; cl2g[h] = 0.69314718056f * cinvg[h];
    }
    float dw[16][4];
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) dw[nt][0] = dw[nt][1] = dw[nt][2] = dw[nt][3] = 0.f;
    double d1[2] = {0.0, 0.0}, d2[2] = {0.0, 0.0};

    for (int jt = 0; jt < ntl; ++jt) {
        const int tile = blockIdx.x + jt * gstep, st = jt % kBStages;
        const int m0 = tile * kPx;
        const uint32_t gks = gk0 + (uint32_t)st * kGkTile, xts = yx0 + (uint32_t)st * kXtTile;
        if (leader && nchunks > 0) {
            bulk_wait_read<0>();                       // the stores of tile jt - 1 have read the staging half
            if (load_existing) {                       // the existing values land in the half while the MMAs run
                mbar_arrive_expect_tx(oload, nchunks * kGkChunk);
                for (int c = 0; c < nchunks; ++c) tma_load_2d(os_u + c * kGkChunk, &p.omap, oload, 64 * wg + 32 * c, m0);
            }
        }
        mbar_wait(smem_u32(&sm.full[st]), (jt / kBStages) & 1);

        // dX^T[in, px] = sum_out W^T[in, out] G[px, out]: 16 k-steps of 8 output channels, N = 32 pixels
        float dx[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) dx[nt][0] = dx[nt][1] = dx[nt][2] = dx[nt][3] = 0.f;
        // dW[out, in] += sum_px G^T[out, px] X[px, in]: 4 k-steps of 8 pixels, N = 128 input channels; A = G^T rows ic, ic + 8
        uint32_t a[4][4];
#pragma unroll
        for (int ks = 0; ks < kPx / 8; ++ks) {
            const int q = 8 * ks + t4;
            a[ks][0] = lds32(gks + kmajor_off(q, ic, kGkChunk)); a[ks][1] = lds32(gks + kmajor_off(q, ic + 8, kGkChunk));
            a[ks][2] = lds32(gks + kmajor_off(q + 4, ic, kGkChunk)); a[ks][3] = lds32(gks + kmajor_off(q + 4, ic + 8, kGkChunk));
        }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 16; ++ks) wgmma_tf32_n32(dx, wa[ks], wgmma_desc(kstep_addr(gks, ks, kGkChunk)));
        wgmma_commit();
#pragma unroll
        for (int ks = 0; ks < kPx / 8; ++ks) wgmma_tf32_n128(dw, a[ks], wgmma_desc(kstep_addr(xts, ks, 0)));
        wgmma_commit();
        warpgroup_bar(2 + wg);                         // the staging half is free (under the MMAs)
        wgmma_wait<1>();                               // the data gradient; the weight-gradient MMAs run on under the epilogue
        wgmma_fence_operand(dx);
        if (load_existing) mbar_wait(oload, jt & 1);

        // ---- epilogue: dx[nt] = {dX^T(ic, px), dX^T(ic, px + 1), dX^T(ic + 8, px), dX^T(ic + 8, px + 1)}, px = 8 nt + 2 t4;
        // pixels >= M and channels >= kin are staged too and clipped by the stores
        float t1[2] = {0.f, 0.f}, t2[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int px = 8 * nt + 2 * t4 + e;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int c = ic + 8 * h;
                    float v = dx[nt][2 * h + e];
                    float *op = reinterpret_cast<float *>(os + kmajor_off(px, icl + 8 * h, kGkChunk));
                    if (load_existing) v += *op;                                    // zeros past M / kin
                    if (final_mode) {
                        // the conversion stored x + half a TF32 ulp (bit pattern + 0x1000, nothing truncated): undo it -> exact fp32 x
                        const float x = __uint_as_float(lds32(xts + kmajor_off(c, px, 0)) - 0x1000u);
                        float em, ls;
                        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(em) : "f"(-1.44269504089f * x));
                        const float sg = 1.f - em;                                  // sigmoid(z) = 1 - exp(-softplus(z))
                        asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(ls) : "f"(fmaxf(sg, 1e-30f)));
                        v *= sg;                                                    // 0 for pixels >= M (G and X are zero there)
                        t1[h] += v;
                        t2[h] = fmaf(v, fmaf(ls, cl2g[h], fmaf(x, cinvg[h], -cbg[h])), t2[h]);
                    }
                    *op = v;
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) { d1[h] += (double)t1[h]; d2[h] += (double)t2[h]; }
        fence_proxy_async();                           // the staged values are read by the TMA stores (async proxy)
        warpgroup_bar(2 + wg);
        if (leader) {
            for (int c = 0; c < nchunks; ++c) {
                if (p.mode == 2) tma_reduce_add_2d(&p.omap, os_u + c * kGkChunk, 64 * wg + 32 * c, m0);
                else tma_store_2d(&p.omap, os_u + c * kGkChunk, 64 * wg + 32 * c, m0);
            }
            bulk_commit();
        }
        wgmma_wait<0>();
        wgmma_fence_operand(a);
        wgmma_fence_operand(dw);
        mbar_arrive(smem_u32(&sm.empty[st]));
    }
    if (final_mode && p.s1) {                          // the four lanes of a channel meet by shuffles
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) {
                d1[h] += __shfl_xor_sync(0xffffffffu, d1[h], o);
                d2[h] += __shfl_xor_sync(0xffffffffu, d2[h], o);
            }
            if (t4 == 0) { atomicAdd(&p.s1[ic + 8 * h], d1[h]); atomicAdd(&p.s2[ic + 8 * h], d2[h]); }
        }
    }
    // flush the weight-gradient accumulators: rows (output channels) ic (+ 8), columns 8 nt + 2 t4 (+ 1)
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
        const int in = 8 * nt + 2 * t4;
        if (in < p.kin) {                              // kin is a multiple of 4: a column pair is inside or outside as a whole
            red_add_v2(p.dW + (size_t)ic * p.lddw + in, dw[nt][0], dw[nt][1]);
            red_add_v2(p.dW + (size_t)(ic + 8) * p.lddw + in, dw[nt][2], dw[nt][3]);
        }
    }
    if (leader) bulk_wait<0>();                        // nothing in flight when the CTA exits
}

}  // namespace

int launch_tc_bwd(const float *dZ, const float *Y, int ldg, const float *ga, const float *m1, const float *m2, const float *mu, const float *rstd,
                  const float *Yprev, int ldp, const float *pa, const float *pb, const float *pmu, const float *prstd, const float *W, int ldw,
                  float *dW, int lddw, float *dZprev, int ldo, int mode, double *s1, double *s2, int M, int kin, int x_raw, cudaStream_t st)
{
    GA_REQUIRE(kin % 4 == 0 && kin >= 4 && kin <= 128 && (!x_raw || mode == 1 || mode == 2), "tensor-core backward: bad kin / mode");
    // the final modes take s1 / s2 over all 128 channels, and mode 3 adds staging chunks that were only loaded below kin
    GA_REQUIRE(kin == 128 || mode == 1 || mode == 2, "tensor-core backward: mode %d needs kin = 128 (kin = %d)", mode, kin);
    GA_REQUIRE(ldg % 4 == 0 && ldp % 4 == 0 && ldw % 4 == 0 && ldo % 4 == 0, "tensor-core backward: leading dimensions must be multiples of 4");
    GA_REQUIRE(lddw % 4 == 0 && (reinterpret_cast<uintptr_t>(dW) & 15) == 0, "tensor-core backward: dW must be 16-byte aligned with lddw a multiple of 4");
    static PerDeviceOnce attr_set;
    if (attr_set.first()) {
        GA_CHECK_CUDA(cudaFuncSetAttribute(tc_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcBwdSmem) + 1024));
    }
    TcBwdParams p{{}, dZ, Y, ldg, ga, m1, m2, mu, rstd, Yprev, ldp, pa, pb, pmu, prstd, W, ldw, dW, lddw, mode, s1, s2, M, kin, x_raw};
    if (int rc = make_tmap(&p.omap, dZprev, kin, M, ldo, kPx)) return rc;
    const int tiles = cdiv(M, kPx), sms = num_sms();
    const int grid = tiles < sms ? tiles : sms;
    {
        ProfScope _ps("mlp_tc_bwd", st);
        tc_bwd_kernel<<<grid, kTcThreads, sizeof(TcBwdSmem) + 1024, st>>>(p);
    }
    GA_CHECK_LAUNCH("tc_bwd_kernel");
    return GA_OK;
}

}  // namespace ga

// Unit-test / building-block entry for the fused backward layer (see tc_bwd_kernel), with every input width the decoder uses.
extern "C" int ga_tc_linear_backward_ex(int32_t M, const float *dZ, const float *Y, int32_t ldg, const float *bwd_coef /*[5][128] ga,m1,m2,mu,rstd or NULL*/,
                                        const float *Yprev, int32_t ldp, const float *prev_coef /*[4][128] a,b,mu,rstd; NULL if x_raw*/, const float *W,
                                        int32_t ldw, float *dW, int32_t lddw, float *dZprev, int32_t ldo, int32_t mode, double *s1, double *s2,
                                        int32_t kin, int32_t x_raw, void *stream)
{
    GA_REQUIRE(M > 0 && dZ && Yprev && (prev_coef || x_raw) && W && dW && dZprev, "bad arguments");
    const float *bc = bwd_coef, *pc = prev_coef;
    return ga::launch_tc_bwd(dZ, Y, ldg, bc, bc ? bc + 128 : nullptr, bc ? bc + 256 : nullptr, bc ? bc + 384 : nullptr, bc ? bc + 512 : nullptr, Yprev,
                             ldp, pc, pc ? pc + 128 : nullptr, pc ? pc + 256 : nullptr, pc ? pc + 384 : nullptr, W, ldw, dW, lddw, dZprev, ldo, mode,
                             s1, s2, M, kin, x_raw, static_cast<cudaStream_t>(stream));
}

// The 128-input-channel, BatchNorm + Softplus input form of the above (the hidden layers).
extern "C" int ga_tc_linear_backward(int32_t M, const float *dZ, const float *Y, int32_t ldg, const float *bwd_coef, const float *Yprev, int32_t ldp,
                                     const float *prev_coef, const float *W, int32_t ldw, float *dW, int32_t lddw, float *dZprev, int32_t ldo,
                                     int32_t mode, double *s1, double *s2, void *stream)
{
    GA_REQUIRE(prev_coef, "bad arguments");
    return ga_tc_linear_backward_ex(M, dZ, Y, ldg, bwd_coef, Yprev, ldp, prev_coef, W, ldw, dW, lddw, dZprev, ldo, mode, s1, s2, 128, 0, stream);
}
