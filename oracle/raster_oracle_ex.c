/*
 * ORACLE — TEST INFRASTRUCTURE ONLY (see raster_oracle_impl.inc and raster_oracle_ex.inc).
 * The original restatement (raster_oracle.c, all of its exports included) plus the SH-colour and precomputed-covariance
 * modes, in both precisions:
 *   oracle32ex_*  REAL=float  — bit-exact target for integer outputs, image / colour reference
 *   oracle64ex_*  REAL=double — gradient reference
 * Build: oracle/raster_oracle_ex.py build() (gcc -O2 -ffp-contract=off -fopenmp, the flags of oracle/Makefile)
 */
#include "raster_oracle.c"

#undef FMA
#undef FMIN
#undef FMAX
#undef SQRT
#undef CEIL
#undef EXP

#define REAL float
#define FN(x) CAT(f32_, x)
#define FMA(a, b, c) fmaf((a), (b), (c))
#define FMIN(a, b) fminf((a), (b))
#define FMAX(a, b) fmaxf((a), (b))
#define SQRT(a) sqrtf(a)
#define CEIL(a) ceilf(a)
#define EXP(a) expf(a)
#include "raster_oracle_ex.inc"
#undef REAL
#undef FN
#undef FMA
#undef FMIN
#undef FMAX
#undef SQRT
#undef CEIL
#undef EXP

#define REAL double
#define FN(x) CAT(f64_, x)
#define FMA(a, b, c) fma((a), (b), (c))
#define FMIN(a, b) fmin((a), (b))
#define FMAX(a, b) fmax((a), (b))
#define SQRT(a) sqrt(a)
#define CEIL(a) ceil(a)
#define EXP(a) exp(a)
#include "raster_oracle_ex.inc"
#undef REAL
#undef FN

enum { QX_RGB = 100, QX_CLAMPED };

/* _get: the original queries on the inner context, plus QX_RGB [P,3] (evaluated or precomputed colour) and QX_CLAMPED [P] */
#define EXPORTS_EX(PFX, V)                                                                                             \
    void *PFX##ex_forward(int P, int H, int W, const float *means3D, const float *colors, const float *opac,            \
                          const float *scales, const float *rots, const float *bg, const float *view, const float *proj,  \
                          float tanfovx, float tanfovy, float scale_modifier, const float *shs, int D, int M,             \
                          const float *campos, const float *cov3D_precomp)                                                \
    {                                                                                                                  \
        return (void *)V##_forward_ex(P, H, W, means3D, colors, opac, scales, rots, bg, view, proj, tanfovx, tanfovy,  \
                                      scale_modifier, shs, D, M, campos, cov3D_precomp);                               \
    }                                                                                                                  \
    long long PFX##ex_num_rendered(void *h) { return (long long)((V##_CtxEx *)h)->c->R; }                              \
    void PFX##ex_free(void *h) { V##_free_ex((V##_CtxEx *)h); }                                                        \
    int PFX##ex_get(void *h, int which, void *dst)                                                                     \
    {                                                                                                                  \
        V##_CtxEx *x = (V##_CtxEx *)h;                                                                                 \
        const size_t P = (size_t)x->c->P;                                                                              \
        if (which == QX_RGB) { PFX##_cpy_real((double *)dst, x->c->colors, 3 * P); return 0; }                         \
        if (which == QX_CLAMPED) { memcpy(dst, x->clamped, P); return 0; }                                             \
        return PFX##_get(x->c, which, dst);                                                                            \
    }                                                                                                                  \
    void PFX##ex_backward(void *h, const float *dL_dout, double *d_mean2D, double *d_conic, double *d_opacity,         \
                          double *d_colors, double *d_means3D, double *d_scales, double *d_rots, double *d_cov3d,       \
                          double *d_sh)                                                                                \
    {                                                                                                                  \
        V##_backward_ex((V##_CtxEx *)h, dL_dout, d_mean2D, d_conic, d_opacity, d_colors, d_means3D, d_scales, d_rots,  \
                        d_cov3d, d_sh);                                                                                \
    }

EXPORTS_EX(oracle32, f32)
EXPORTS_EX(oracle64, f64)
