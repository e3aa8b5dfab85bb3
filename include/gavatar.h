/*
 * gavatar.h — C ABI of libgavatar_sm90.so, the H100-native (sm_90a) implementation of GaussianAvatar's per-frame
 * render hot path.  Flat extern "C" surface: plain device/host pointers, sizes, a CUDA stream handle passed as
 * void*.  No torch types.  Every function returns 0 (GA_OK) or a negative GaStatus; ga_last_error() gives the
 * message of the last failure on the calling thread.  The library never allocates persistent device memory: the
 * caller owns every buffer (sizes from the *_bytes queries) and keeps them alive until the matching backward ran.
 *
 * All work is enqueued on `stream`; calls are asynchronous unless stated otherwise.  Not re-entrant per workspace;
 * independent workspaces / streams may run concurrently.  One process per GPU.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference; [UPSTREAM] = the un-vendored
 * diff-gaussian-rasterization extension the reference imports at gaussian_renderer/__init__.py:6):
 *
 *   ga_raster_*          GaussianRasterizer(raster_settings)(means3D=..., ...)      gaussian_renderer/__init__.py:36-48
 *                        ([UPSTREAM] _C.rasterize_gaussians / _C.rasterize_gaussians_backward)
 *   ga_lbs_*             pred_res*0.02 / mask-select / +query_points / two einsums / scale ramp / repeat / reg. losses
 *                                                                                    model/avatar_model.py:308-330
 *   ga_smpl_*            SMPL.forward(...).A @ inv_mats                              model/avatar_model.py:291-296,
 *                                                                                    submodules/smplx/lbs.py:152-252,349-405
 *   ga_decoder_* ga_conv* POP_no_unet.forward (GeomConvLayers, grid_sample, ShapeDecoder)
 *                                                                                    model/network.py:39-83, model/modules.py:114-137,508-582
 *   ga_loss_*            l1_loss_w + ssim                                            utils/loss_utils.py:7-53
 *   ga_adam_*            torch.optim.Adam step on net + geo_feature                  model/avatar_model.py:148-155,264-267
 *   ga_lpips_*           lpips.LPIPS(net='alex')((image-0.5)*2, (gt_image-0.5)*2)     train.py:26,89-91
 *   ga_metrics_*         torchmetrics PeakSignalNoiseRatio / StructuralSimilarityIndexMeasure  eval.py:12,20-35
 */
#ifndef GAVATAR_H_
#define GAVATAR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum GaStatus {
    GA_OK = 0,
    GA_ERR_INVALID = -1,   /* bad shape / null pointer / unsupported option */
    GA_ERR_CAPACITY = -2,  /* a caller-provided buffer is too small */
    GA_ERR_CUDA = -3       /* a CUDA runtime call failed; see ga_last_error() */
} GaStatus;

int ga_version(void);
const char *ga_last_error(void);
/* Number of kernels this library has launched in the calling process since load (bench.py's gpu_launches). */
long long ga_launch_count(void);
/* Optional per-kernel CUDA-event timing of this library's launches (bench.py roofline leg).  ga_profile_report
 * synchronises the device and writes one "name count total_ms" line per kernel name, then clears the log. */
void ga_profile_enable(int on);
int ga_profile_report(char *buf, size_t cap);

/* ------------------------------------------------------------------------------------------------------------------
 * Rasterizer.  Layout contracts (SURVEY.md §8b): contiguous fp32; means3D [P,3]; colors [P,3] (colors_precomp);
 * opacities [P]; scales [P,3]; rotations [P,4] (w,x,y,z, un-normalised); bg [3]; viewmatrix / projmatrix = the
 * reference's transposed 4x4s (scene/dataset_mono.py:248-250), i.e. flat[col*4+row]; image planar [3,H,W];
 * radii int32 [P].
 * ---------------------------------------------------------------------------------------------------------------- */
/* Antialiasing (upstream's `antialiasing` setting, Mip-Splatting's screen-space filter), one flag per Gaussian set: 0 renders
 * with the fixed 0.3 px^2 dilation alone, as upstream without the setting; nonzero also scales each splat's opacity so that its
 * footprint integrates to what the undilated Gaussian's would.  With Sigma2 = [[a0, b], [b, c0]] the projected 2D covariance
 * before the dilation, a = a0 + 0.3 and c = c0 + 0.3 (conic, radius and tile rect come from (a, b, c) either way):
 *   r = (a0 c0 - b^2) / (a c - b^2),   rho = sqrt(max(2.5e-5, r)),   stored opacity (conic_opacity w) = o rho.
 * Nothing else changes: radii, rects, depths, xy, conics and the binning are the call without it's, bit for bit.  The backwards
 * return dL/do = gO rho (gO: dL/d of the stored opacity) and, where r > 2.5e-5, add gO o / (2 rho) dr/d(a0, b, c0) to the 2D
 * covariance gradients; they recover o as the stored opacity over rho recomputed from their own covariance, so a backward must
 * be given the flag its forward had. */
typedef struct GaRasterSettings {
    int32_t P, H, W;
    float tanfovx, tanfovy, scale_modifier;
    int32_t antialiasing;        /* 0: off (zero-initialised settings behave as before), else on; see above     */
} GaRasterSettings;

size_t ga_raster_geom_bytes(int32_t P);                       /* per-Gaussian state (upstream's geomBuffer)   */
size_t ga_raster_img_bytes(int32_t H, int32_t W);             /* final_T, n_contrib, tile ranges / counts, status (imgBuffer) */
size_t ga_raster_binning_bytes(int64_t num_rendered, int32_t H, int32_t W); /* tile buckets, sorted list, packed records, checkpoints (binningBuffer) */
size_t ga_raster_bwd_scratch_bytes(int32_t P);                /* dL/dmean2D, dL/dconic, dL/dopacity scratch   */

/* Per-frame API, upstream's call shape (the host sizes the binning buffer from the instance count).
 * Stage 1: K1 preprocess (+ per-tile instance counts) and the tile scan.  Synchronises `stream` once to return the number of
 * (Gaussian, tile) instances (upstream does the same D2H read to size its binning buffer). */
int ga_raster_forward_preprocess(const GaRasterSettings *s, const float *means3D, const float *scales,
                                 const float *rotations, const float *opacities, const float *viewmatrix,
                                 const float *projmatrix, void *geom, void *img, int32_t *radii, int64_t *num_rendered_host,
                                 void *stream);
/* Stage 2: K3 scatter into tile buckets, K4 per-tile sort (upstream's order: depth bits, then Gaussian index), K6 alpha
 * compositing.  `binning` must hold ga_raster_binning_bytes(num_rendered, H, W). */
int ga_raster_forward_render(const GaRasterSettings *s, const float *colors, const float *bg, void *geom, void *binning,
                             size_t binning_bytes, int64_t num_rendered, void *img, float *out_color, void *stream);
/* Backward (K7 + fused K8/K9).  d_opacities, d_rotations, d_means2D ([P,3], xy filled) may be NULL.
 * d_* outputs are overwritten (not accumulated). */
int ga_raster_backward(const GaRasterSettings *s, const float *means3D, const float *colors, const float *scales,
                       const float *rotations, const float *bg, const float *viewmatrix, const float *projmatrix,
                       const int32_t *radii, const void *geom, const void *binning, const void *img,
                       int64_t num_rendered, const float *dL_dout, void *scratch, float *d_means3D, float *d_colors,
                       float *d_scales, float *d_rotations, float *d_opacities, float *d_means2D, void *stream);

/* The other colour and covariance inputs of upstream's API (per-frame path only).
 * SH colours: rgb = max(sum_k basis_k(dir) shs[k] + 0.5, 0) per channel, dir = (mean - campos) / |mean - campos|, evaluated in
 * stage 1 for the Gaussians that survive the culls into `rgb` (then passed as `colors` to ga_raster_forward_render), with the
 * clamped channels recorded in `clamped` for the backward.  Precomputed covariances replace scales / rotations / scale_modifier. */
typedef struct GaRasterColorCov {
    const float *shs;            /* [P, sh_coeffs, 3] or NULL: colours are precomputed                     */
    int32_t sh_degree, sh_coeffs;/* active degree 0..3; coefficients per Gaussian >= (sh_degree + 1)^2    */
    const float *campos;         /* [3] device; required with shs                                          */
    const float *cov3D_precomp;  /* [P, 6] (xx, xy, xz, yy, yz, zz) or NULL: Sigma from scales / rotations */
    float *rgb;                  /* [P, 3] written by the forward, read by the backward (with shs)         */
    uint8_t *clamped;            /* [P] bit c = channel c clamped (with shs)                               */
} GaRasterColorCov;
/* ga_raster_forward_preprocess with a colour / covariance descriptor (cc NULL: identical to it).  scales / rotations may be NULL
 * with cov3D_precomp. */
int ga_raster_forward_preprocess_ex(const GaRasterSettings *s, const GaRasterColorCov *cc, const float *means3D,
                                    const float *scales, const float *rotations, const float *opacities,
                                    const float *viewmatrix, const float *projmatrix, void *geom, void *img, int32_t *radii,
                                    int64_t *num_rendered_host, void *stream);
/* ga_raster_backward with the same descriptor as the forward (cc NULL: identical to it).  With shs: colors may be NULL, d_colors
 * receives dL/drgb before the clamp mask, and d_sh [P, sh_coeffs, 3] is overwritten (0 for k >= (sh_degree + 1)^2, clamped
 * channels and culled Gaussians); the direction term is included in d_means3D.  With cov3D_precomp: d_cov3D [P, 6] receives
 * dL/dSigma (an off-diagonal entry stands for both symmetric entries); scales, rotations, d_scales, d_rotations may be NULL and are
 * not written. */
int ga_raster_backward_ex(const GaRasterSettings *s, const GaRasterColorCov *cc, const float *means3D, const float *colors,
                          const float *scales, const float *rotations, const float *bg, const float *viewmatrix,
                          const float *projmatrix, const int32_t *radii, const void *geom, const void *binning, const void *img,
                          int64_t num_rendered, const float *dL_dout, void *scratch, float *d_means3D, float *d_colors,
                          float *d_scales, float *d_rotations, float *d_opacities, float *d_means2D, float *d_sh, float *d_cov3D,
                          void *stream);

/* Batched API: the B <= 8 frames a training step renders (model/avatar_model.py:332-365 loops them) in ONE set of launches
 * and WITHOUT any host read-back, so a whole step can be captured in a CUDA graph.  All frames share H, W and P.
 * Arrays are [B,P,*] (rotations / opacities: [P,*] shared by every frame when the stride is 0); out_color [B,3,H,W];
 * radii [B,P]; cams [B,40] device floats per frame: viewmatrix 0..15, projmatrix 16..31 (the reference's transposed 4x4s),
 * tanfovx 32, tanfovy 33, camera centre 34..36 (read by ga_rasterb_forward_scene only).  `capacity` = number of (Gaussian, tile) instances the caller sized `binning` for; if a step needs
 * more, status[1] is set, the tiles that do not fit are rendered as empty and nothing is overrun — the caller re-runs with a
 * larger buffer (status[0] = the count needed).  status (device, 16 x int32, inside `img`): [0] instances, [1] overflow,
 * [2] backward segments, [4+b] first instance of frame b, [4+B] = [0]. */
typedef struct GaRasterBatchDesc {
    int32_t B, P, H, W;
    int64_t capacity;
    int64_t rot_stride, opac_stride;   /* floats between two frames' rotations / opacities: 4P / P, or 0 = shared */
    float scale_modifier;
    int32_t antialiasing;              /* of the dynamic set (see GaRasterSettings); a backward takes its forward's */
} GaRasterBatchDesc;
size_t ga_rasterb_geom_bytes(int32_t B, int32_t P);
size_t ga_rasterb_img_bytes(int32_t B, int32_t H, int32_t W);
size_t ga_rasterb_binning_bytes(int32_t B, int32_t H, int32_t W, int64_t capacity);
size_t ga_rasterb_bwd_scratch_bytes(int32_t B, int32_t P);
const int32_t *ga_rasterb_status(int32_t B, int32_t H, int32_t W, const void *img);   /* device pointer of the status words */
/* Copy the 16 status words to PINNED host memory behind the latest forward (asynchronous, capturable in a CUDA graph); word 15
 * receives *serial_dev (device int32 the caller bumps before every forward) so the host can tell which forward a copy is of. */
int ga_rasterb_status_to_host(int32_t B, int32_t H, int32_t W, void *img, const int32_t *serial_dev, int32_t *host16_pinned,
                              void *stream);
int ga_rasterb_forward(const GaRasterBatchDesc *d, const float *cams, const float *bg, const float *means3D,
                       const float *colors, const float *scales, const float *rotations, const float *opacities, void *geom,
                       void *img, void *binning, int32_t *radii, float *out_color, void *stream);
/* d_rotations [B,P,4], d_opacities [B,P] and d_means2D [B,P,3] (each may be NULL) are written per frame whatever rot_stride /
 * opac_stride are: with shared rotations / opacities the caller sums the frames. */
int ga_rasterb_backward(const GaRasterBatchDesc *d, const float *cams, const float *bg, const float *means3D,
                        const float *colors, const float *scales, const float *rotations, const int32_t *radii,
                        const void *geom, const void *img, const void *binning, const float *dL_dout, void *scratch,
                        float *d_means3D, float *d_colors, float *d_scales, float *d_rotations, float *d_opacities,
                        float *d_means2D, void *stream);

/* A static Gaussian set for ga_rasterb_forward_scene: a 3D Gaussian Splatting scene shared by every frame (read with frame stride
 * 0, never copied per frame).  Its colours are spherical harmonics, evaluated for each frame's camera centre exactly as
 * GaRasterColorCov's are: rgb = max(sum_k basis_k(dir) shs[k] + 0.5, 0), dir = (mean - campos) / |mean - campos|, 0 for Gaussians
 * the frame culls.  Forward only: there is no backward of the composite. */
typedef struct GaRasterScene {
    int32_t Ps;                  /* static Gaussians (0: the composite renders the dynamic set alone)        */
    int32_t sh_degree, sh_coeffs;/* active degree 0..3; coefficients per Gaussian >= (sh_degree + 1)^2     */
    const float *means3D;        /* [Ps, 3]                                                                 */
    const float *scales;         /* [Ps, 3] activated (times the descriptor's scale_modifier, as the dynamic set) */
    const float *rotations;      /* [Ps, 4] (w, x, y, z), normalised                                        */
    const float *opacities;      /* [Ps] activated                                                          */
    const float *shs;            /* [Ps, sh_coeffs, 3]                                                      */
    float *rgb;                  /* [B, Ps, 3] written: frame b's evaluated colours                         */
    int32_t antialiasing;        /* of the static set (see GaRasterSettings), independent of the dynamic set's */
} GaRasterScene;
/* ga_rasterb_forward of the dynamic set (d->P, arrays and strides as there) splatted together with a static scene set in one sort
 * per tile, so that each occludes the other correctly.  Frame b has P + Ps Gaussians, the dynamic P first, then the static set:
 * that order fixes radii [B, P+Ps], geom (sized by ga_rasterb_geom_bytes(B, P + Ps)), ga_raster_views(B, P + Ps, ...) and
 * upstream's tie order (depth bits, then index).  cams rows must carry the camera centre in words 34..36 (upstream's `campos`).
 * Binning, the capacity / overflow status and compositing are ga_rasterb_forward's. */
int ga_rasterb_forward_scene(const GaRasterBatchDesc *d, const GaRasterScene *scene, const float *cams, const float *bg,
                             const float *means3D, const float *colors, const float *scales, const float *rotations,
                             const float *opacities, void *geom, void *img, void *binning, int32_t *radii, float *out_color,
                             void *stream);

/* Index ranges of the dynamic set for ga_rasterb_forward_mattes, e.g. several avatars concatenated into one [B, P1+...+PK, *]
 * set.  Entry idx of a frame belongs to set k when first[k] <= idx < first[k+1]; indices at or above first[K] (the rest of the
 * dynamic set, and the scene's) belong to no set. */
typedef struct GaRasterSets {
    int32_t K;                   /* 1..8 sets                                                               */
    int32_t first[9];            /* first[0] = 0, nondecreasing up to first[K] <= d->P; entries past K unread */
    float *mattes;               /* [B, K, H, W] written                                                    */
} GaRasterSets;
/* ga_rasterb_forward_scene (scene NULL or Ps = 0: ga_rasterb_forward of the dynamic set alone) that also writes, for each set
 * and pixel, the weight its Gaussians added to the pixel: matte_k = sum over set k's blended entries of alpha T, the same
 * weights the colour is blended with, so sum_k matte_k = 1 - final T where every entry belongs to a set.  Binning, the capacity
 * / overflow status, tie order and every other output are the composite's, bit for bit.  Bad K or first, or a NULL mattes,
 * are refused before anything launches.  Forward only. */
int ga_rasterb_forward_mattes(const GaRasterBatchDesc *d, const GaRasterScene *scene, const GaRasterSets *sets, const float *cams,
                              const float *bg, const float *means3D, const float *colors, const float *scales,
                              const float *rotations, const float *opacities, void *geom, void *img, void *binning,
                              int32_t *radii, float *out_color, void *stream);
/* ga_rasterb_forward_mattes (sets NULL: no mattes; scene NULL or Ps = 0: no scene) that also writes a depth pass, depth
 * [B, 2, H, W] fp32, over the entries each pixel blends, with the weights w_i = alpha_i T_i its colour uses.  z_i is the entry's
 * view-space depth in world units (the scene's units after its placement; K1 culls z <= 0.2, so 0 means no surface):
 *   plane 0, mean depth:   D / (1 - T) with D = sum_i w_i z_i (accumulated as the colour channels are, so D is bit for bit the
 *                          red channel a colour (z_i, 0, 0) with bg = 0 gives) and T the final transmittance; 0 where n_contrib = 0;
 *   plane 1, median depth: z of the first blended entry after which T <= 0.5; 0 where the final T > 0.5.
 * Every other output (and the mattes, with sets) is the call without depth's, bit for bit.  A NULL depth, or bad sets when sets
 * are given, are refused before anything launches.  Forward only. */
int ga_rasterb_forward_depth(const GaRasterBatchDesc *d, const GaRasterScene *scene, const GaRasterSets *sets, float *depth,
                             const float *cams, const float *bg, const float *means3D, const float *colors, const float *scales,
                             const float *rotations, const float *opacities, void *geom, void *img, void *binning, int32_t *radii,
                             float *out_color, void *stream);

/* Training against depth maps: ga_rasterb_forward / ga_rasterb_backward with the mean depth differentiable.
 * ga_rasterb_forward_depth_train is ga_rasterb_forward_depth of the dynamic set alone (no scene, no sets): images, radii, every
 * buffer and both depth planes are that call's, bit for bit.  It also fills `depth_state` (ga_rasterb_depth_state_bytes(B, H, W,
 * capacity), caller-owned, to be kept with geom / img / binning until the backward): each pixel's D = sum_i w_i z_i at the start of
 * every 256-entry segment of its tile's list and at its end, where z_i is the entry's view-space z in world units (the z K1 culls at
 * 0.2 and sorts by, not the length of the ray) and w_i = alpha_i T_i.  A depth_state smaller than the size query asks is refused
 * with GA_ERR_CAPACITY; NULL pointers are refused; both before anything launches.
 *
 * ga_rasterb_backward_depth is ga_rasterb_backward plus the gradient of dL_ddepth [B,H,W] = dL/dm, m = D / A the mean depth
 * (plane 0 of that forward's `depth`, passed back unchanged), A = 1 - T_final:
 *   dL/dz_i     = (g / A) w_i
 *   dL/dalpha_i += (g / A) [T_i (z_i - zhat_i) - m T_final / (1 - alpha_i)],  zhat_i the depth composited behind entry i
 * (un-premultiplied; a segment starts from the stored D: zhat = (D_final - D_ckpt) / T_ckpt).  dL/dalpha flows through the
 * conic / mean2D / opacity chain as the colour's does; dL/dz enters d_means3D through the view matrix's z row.  Plane 1 (the
 * median) is not differentiated.  scratch: ga_rasterb_depth_bwd_scratch_bytes(B, P) bytes (d_mean2D, d_conic_op as for
 * ga_rasterb_backward, then dL/dz [B,P]).  Undersized depth_state or scratch and NULL pointers are refused before any launch. */
size_t ga_rasterb_depth_state_bytes(int32_t B, int32_t H, int32_t W, int64_t capacity);
size_t ga_rasterb_depth_bwd_scratch_bytes(int32_t B, int32_t P);
int ga_rasterb_forward_depth_train(const GaRasterBatchDesc *d, float *depth, void *depth_state, size_t depth_state_bytes,
                                   const float *cams, const float *bg, const float *means3D, const float *colors, const float *scales,
                                   const float *rotations, const float *opacities, void *geom, void *img, void *binning, int32_t *radii,
                                   float *out_color, void *stream);
int ga_rasterb_backward_depth(const GaRasterBatchDesc *d, const float *cams, const float *bg, const float *means3D,
                              const float *colors, const float *scales, const float *rotations, const int32_t *radii,
                              const void *geom, const void *img, const void *binning, const float *dL_dout, const float *dL_ddepth,
                              const float *depth, const void *depth_state, size_t depth_state_bytes, void *scratch,
                              size_t scratch_bytes, float *d_means3D, float *d_colors, float *d_scales, float *d_rotations,
                              float *d_opacities, float *d_means2D, void *stream);

/* Debug / parity accessors into the opaque buffers (device pointers; valid after the forward that filled them).  B = 1 and
 * capacity = num_rendered for buffers of the per-frame API. */
typedef struct GaRasterViews {
    const float *depth;          /* [B*P]   */
    const float *xy;             /* [B*P,2] */
    const float *conic_opacity;  /* [B*P,4] */
    const float *cov3d;          /* [B*P,6] */
    const uint32_t *tiles_touched; /* [B*P] */
    const uint16_t *rect;        /* [B*P,4] min.x min.y max.x max.y */
    const uint32_t *point_list;  /* [R] Gaussian indices, tile by tile, in upstream's sorted order */
    const uint32_t *ranges;      /* [B*T,2] [start,end) into point_list (frame b starts at status[4+b]) */
    const uint32_t *tile_count;  /* [B*T] */
    const float *final_T;        /* [B*H*W] */
    const uint32_t *n_contrib;   /* [B*H*W] */
    const int32_t *status;       /* [16] */
} GaRasterViews;
int ga_raster_views(int32_t B, int32_t P, int32_t H, int32_t W, int64_t capacity, const void *geom, const void *binning,
                    const void *img, GaRasterViews *out);

/* ------------------------------------------------------------------------------------------------------------------
 * SMPL joint transforms -> cano2live (model/avatar_model.py:291-296; submodules/smplx/lbs.py:299-405;
 * body_models.py:380-383).  pose [B,72] axis-angle, transl [B,3], rest_joints [24,3] (J_regressor (v_template +
 * shapedirs beta), constant per subject), inv_cano [24,4,4] = inv(A_cano) -> cano2live [B,24,12] (3x4 row-major per
 * joint).  saved_G [B,24,12] is kept by the caller for the backward.
 * ---------------------------------------------------------------------------------------------------------------- */
int ga_smpl_forward(int32_t B, const float *pose, const float *transl, const float *rest_joints, const float *inv_cano,
                    float *cano2live, float *saved_G, void *stream);
int ga_smpl_backward(int32_t B, const float *pose, const float *rest_joints, const float *inv_cano, const float *saved_G,
                     const float *d_cano2live, float *d_pose, float *d_transl, void *stream);
/* SMPL-X (55 joints: global, 21 body, jaw, left / right eye, 15 left-hand, 15 right-hand).  pose [B,66] holds the 22 trainable
 * joints, rest_pose [B,99] the other 33 (model/avatar_model.py:279-289; flat_hand_mean=True, no PCA, no expression).
 * rest_joints [55,3], inv_cano [55,4,4] -> cano2live [B,55,12]; saved_G [B,55,12].  The backward writes d_pose [B,66] and
 * d_transl [B,3]; rest_pose gets no gradient. */
int ga_smplx_forward(int32_t B, const float *pose, const float *rest_pose, const float *transl, const float *rest_joints,
                     const float *inv_cano, float *cano2live, float *saved_G, void *stream);
int ga_smplx_backward(int32_t B, const float *pose, const float *rest_pose, const float *rest_joints, const float *inv_cano,
                      const float *saved_G, const float *d_cano2live, float *d_pose, float *d_transl, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Stage-2 input position maps (scripts/gen_pose_map_our_smpl.py: smplx forward, then PosRender in UV space).
 *
 * ga_smpl_vertices: posed SMPL mesh vertices of B <= 8 frames (submodules/smplx/lbs.py:lbs vertices + body_models.py:380-382):
 *   verts[b] = sum_j w_vj A_j(b) [v_shaped + posedirs^T (R_j(b) - I)_{j=1..23}; 1] + transl[b].  pose [B,72], transl [B,3],
 *   rest_joints [24,3], v_shaped [V,3] = v_template + shapedirs beta (constant per subject), posedirs [207, 3V] (the layout the
 *   reference's smplx.SMPL keeps), weights [V,24] -> verts [B,V,3].  posedirs is read once per call for all B frames.
 * ga_posmap_layout: which face covers each texel of an S x S map (1 <= S <= 512) and with which barycentric weights, from the UV
 *   corners of every face uv_corners [F,3,2] (uv[faces_uv]).  face_id [S,S] int32 (-1: no face; the reference's
 *   uv_mask{S}_with_faceid_smpl.npy format), bary [S,S,3].  Output row r, column c samples u = (c+0.5)/S, v = 1-(r+0.5)/S.
 *   Coverage is exact integer arithmetic on coordinates snapped to 1/256 texel, lowest face index wins; the rules are in
 *   csrc/posmap.cu and DESIGN.md.  Run once per (template, S).
 * ga_posmap_fill: out [B,3,S,S] = sum_i bary_i verts[b, faces[face_id, i]] (0 where face_id is -1); faces [F,3] int32 must index
 *   vertices below V and face_id must come from ga_posmap_layout over the same F faces.  Every element of `out` is written.
 * ---------------------------------------------------------------------------------------------------------------- */
int ga_smpl_vertices(int32_t B, int32_t V, const float *pose, const float *transl, const float *rest_joints, const float *v_shaped,
                     const float *posedirs, const float *weights, float *verts, void *stream);
/* ga_smplx_vertices: the SMPL-X counterpart of ga_smpl_vertices (smplx.SMPLX(use_pca=False, flat_hand_mean=True) vertices +
 *   transl, body_models.py:1273-1275): pose [B,66] (global + 21 body joints), rest_pose [B,99] (jaw, left / right eye, 15 + 15
 *   finger joints), transl [B,3], rest_joints [55,3], v_shaped [V,3], posedirs [486, 3V], weights [V,55] -> verts [B,V,3], B <= 8.
 *   posedirs is read once per call for all B frames, and a frame's result does not depend on the batch it is in.
 * ga_posmap_weights: the texel skinning-weight map out [S,S,J] = sum_i bary_i weights[faces[face_id, i], :] (0 where face_id is
 *   -1), J = 24 or 55; weights [V,J], faces [F,3] int32 indexing vertices below V, face_id / bary from ga_posmap_layout over the
 *   same F faces (utils/general_utils.py:245-259, the lbs_map_{body}_{S}.npy format).  Every element of `out` is written. */
int ga_smplx_vertices(int32_t B, int32_t V, const float *pose, const float *rest_pose, const float *transl, const float *rest_joints,
                      const float *v_shaped, const float *posedirs, const float *weights, float *verts, void *stream);
int ga_posmap_weights(int32_t S, int32_t J, const float *weights, const int32_t *faces, const int32_t *face_id, const float *bary,
                      float *out, void *stream);
int ga_posmap_layout(int32_t F, int32_t S, const float *uv_corners, int32_t *face_id, float *bary, void *stream);
int ga_posmap_fill(int32_t B, int32_t S, int32_t V, const float *verts, const int32_t *faces, const int32_t *face_id,
                   const float *bary, float *out, void *stream);

/* Gradients of the position maps with respect to pose and transl (test-time pose fitting through a stage-2 avatar).
 *
 * ga_smpl_vertices_backward / ga_smplx_vertices_backward: the adjoints of ga_smpl_vertices / ga_smplx_vertices.  From the forward's
 *   inputs (transl does not enter the gradient) and d_verts [B,V,3] they write d_pose [B,72] (SMPL) or [B,66] (SMPL-X) and d_transl
 *   [B,3], through both the pose blend shapes (posedirs, R_j - I) and the skinning transforms A_j (the joint chain).  SMPL-X's
 *   rest_pose [B,99] is data and has no gradient.  1 <= B <= 8; posedirs is read once per call for all frames.  workspace:
 *   ga_*_vertices_backward_workspace_bytes(B, V) bytes, 4-byte aligned, scratch of the call (per-CTA partial sums, added in a fixed
 *   order by a second kernel).  No floating-point atomics: the results are bit-reproducible and a frame's do not depend on the batch.
 * ga_posmap_vertex_csr: for the layout face_id [S,S] of faces [F,3] (indices below V), the vertex -> (texel, corner) lists the fill
 *   backward runs over: offsets [V+1] and entries [3 S^2] (int32; the first offsets[V] are used), entry 3 t + i for texel t whose
 *   covering face has the vertex as corner i, ascending within each vertex.  Run once per layout.
 * ga_posmap_fill_backward: d_verts [B,V,3] = sum over each vertex's entries of bary[t,i] d_out[b,:,t], for d_out [B,3,S,S], 1 <= B <= 8.
 *   No atomics; every element of d_verts is written (0 for a vertex no texel uses). */
size_t ga_smpl_vertices_backward_workspace_bytes(int32_t B, int32_t V);
size_t ga_smplx_vertices_backward_workspace_bytes(int32_t B, int32_t V);
int ga_smpl_vertices_backward(int32_t B, int32_t V, const float *pose, const float *rest_joints, const float *v_shaped,
                              const float *posedirs, const float *weights, const float *d_verts, void *workspace, size_t workspace_bytes,
                              float *d_pose, float *d_transl, void *stream);
int ga_smplx_vertices_backward(int32_t B, int32_t V, const float *pose, const float *rest_pose, const float *rest_joints,
                               const float *v_shaped, const float *posedirs, const float *weights, const float *d_verts, void *workspace,
                               size_t workspace_bytes, float *d_pose, float *d_transl, void *stream);
int ga_posmap_vertex_csr(int32_t S, int32_t V, const int32_t *faces, const int32_t *face_id, int32_t *offsets, int32_t *entries,
                         void *stream);
int ga_posmap_fill_backward(int32_t B, int32_t S, int32_t V, const int32_t *csr_offsets, const int32_t *csr_entries, const float *bary,
                            const float *d_out, float *d_verts, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Fused Gaussian LBS + attribute assembly (model/avatar_model.py:308-326).  dec_out [S*S,8] pixel-major packed decoder
 * output (res.xyz, scale, rgb, pad); valid_index [N] int32 = flat UV index of the n-th valid pixel; query_points [N,3];
 * query_lbs [N,24]; cano2live [B,24,12]; scale_mul = 1e-3*iteration if iteration<1000 else 1 (avatar_model.py:316-319).
 * Outputs per frame in the rasterizer's layout: means3D / scales3 / colors [B,N,3].  B <= 8.
 * Backward overwrites d_dec_out [num_pixels,8] (zero at invalid pixels) and d_cano2live [B,24,12].
 * ---------------------------------------------------------------------------------------------------------------- */
int ga_lbs_forward(int32_t N, int32_t B, float scale_mul, int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index,
                   const float *query_points, const float *query_lbs, const float *cano2live, float *means3D,
                   float *scales3, float *colors, void *stream);
/* dec_frame_stride: floats between two frames' decoder outputs — 0 in stage 1 (ONE [S*S,8] output serves every frame and the
 * backward SUMS the frames' gradients into d_dec_out [num_pixels,8]), S*S*8 in stage 2 (per-frame outputs, model/avatar_model.py:
 * 401-420; d_dec_out is then [B*S*S,8] and num_pixels = B*S*S). */
int ga_lbs_backward(int32_t N, int32_t B, int32_t num_pixels, float scale_mul, int64_t dec_frame_stride, const float *dec_out,
                    const int32_t *valid_index, const float *query_points, const float *query_lbs, const float *cano2live,
                    const float *d_means3D, const float *d_scales3, const float *d_colors, float *d_dec_out,
                    float *d_cano2live, void *stream);
/* The same for either body model: num_joints 24 (SMPL) or 55 (SMPL-X); query_lbs is [N, lbs_ld] with lbs_ld a multiple of 4 and
 * >= num_joints (the columns past num_joints are ignored); cano2live / d_cano2live are [B, num_joints, 12].  Built layouts:
 * (24, 24) and (55, 56); ga_lbs_forward / ga_lbs_backward are the (24, 24) case. */
int ga_lbs_forward_ex(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, float scale_mul, int64_t dec_frame_stride,
                      const float *dec_out, const int32_t *valid_index, const float *query_points, const float *query_lbs,
                      const float *cano2live, float *means3D, float *scales3, float *colors, void *stream);
int ga_lbs_backward_ex(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, int32_t num_pixels, float scale_mul,
                       int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index, const float *query_points,
                       const float *query_lbs, const float *cano2live, const float *d_means3D, const float *d_scales3,
                       const float *d_colors, float *d_dec_out, float *d_cano2live, void *stream);
/* The same with each training frame's exposure: frame b's colours become c' = A c + t, [A | t] = exposure[pose_idx[b]] (row-major
 * 3x4 per row, exposure [num_exposures,12], pose_idx [B] int32, both in device memory: nothing is read on the host).  A frame whose
 * pose_idx is outside [0, num_exposures) gets NaN colours.  Means and scales are those of ga_lbs_forward_ex.  The backward also
 * writes d_exposure [num_exposures,12]: row f is the sum, over the frames with pose_idx == f in slot order, of
 * sum_n g_n (x) [c_n, 1] (g the colour gradient, c the decoder colour); rows no frame touches and row 0 (the gauge anchor) are 0.
 * No atomics reach d_exposure: equal inputs give equal bits.  Its decoder colour gradient is A^T g; d_cano2live is that of
 * ga_lbs_backward_ex.  workspace: at least ga_lbs_exposure_workspace_bytes(N, num_joints) bytes of device memory. */
size_t ga_lbs_exposure_workspace_bytes(int32_t N, int32_t num_joints);
int ga_lbs_forward_exposure(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, float scale_mul, int64_t dec_frame_stride,
                            const float *dec_out, const int32_t *valid_index, const float *query_points, const float *query_lbs,
                            const float *cano2live, int32_t num_exposures, const float *exposure, const int32_t *pose_idx,
                            float *means3D, float *scales3, float *colors, void *stream);
int ga_lbs_backward_exposure(int32_t N, int32_t B, int32_t num_joints, int32_t lbs_ld, int32_t num_pixels, float scale_mul,
                             int64_t dec_frame_stride, const float *dec_out, const int32_t *valid_index, const float *query_points,
                             const float *query_lbs, const float *cano2live, int32_t num_exposures, const float *exposure,
                             const int32_t *pose_idx, const float *d_means3D, const float *d_scales3, const float *d_colors,
                             float *d_dec_out, float *d_cano2live, float *d_exposure, void *workspace, size_t workspace_bytes,
                             void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Stage-1 feature net (model/network.py:39-83; model/modules.py:114-137,508-582,745-754): geometry convs -> bilinear
 * UV up-sampling -> [features | uv] -> ShapeDecoder with training-mode BatchNorm.  Parameters live in ONE flat fp32
 * buffer (offsets from ga_decoder_layout, in floats; kernel-friendly packing):
 *   gconv[i]   [25][64][64]  (tap, c_in, c_out)          <- geom_proc_layers.conv{i+1}.weight [co,ci,5,5]
 *   w[0]       [128][72]     conv1, input padded 66->72   w[1..3] [128][128] conv2..4
 *   w[4]       [128][200]    conv5 over [feat(72) | x4(128)]
 *   w[5]       [384][128]    conv6, conv6N, conv6SH stacked; w[6] [3][128][128] conv7, conv7N, conv7SH
 *   b/gamma/beta[l]  bias and BatchNorm affine of the same layers (head order xyz, N, SH)
 *   w8 [8][128]  rows conv8 (3), conv8N (1), conv8SH (3), zero row;  b8 [8]
 * geo_nchw is `geo_feature` [1,64,feat_res,feat_res]; bn_running [2][1408] running mean / var (nullable);
 * dec_out [S*S, 8] = (res.xyz, scale, rgb, 0).  The workspace keeps every activation for the backward.
 * `batch` only enters the unbiased running-variance update: stage-1 inputs are identical across the batch, so the net
 * is evaluated once per step (SURVEY.md §8 a-4) and d_dec_out must already be summed over the frames.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct GaDecoderDesc {
    int32_t S, feat_res, batch, c_geom, hsize;
    float bn_eps, bn_momentum;
    int32_t flags;   /* GA_DECODER_TENSOR_CORES: MLP layers on the tensor cores (TF32, the reference's cuDNN numerics); 0: strict FP32 */
    int32_t frames;  /* distinct input maps = decoder row blocks: 0 / 1 = stage 1 (one map shared by the batch), B = stage 2 (one
                      * pose_featmap per frame, model/avatar_model.py:401-405): rows, dec_out and d_dec_out are then [frames*S*S, .] */
} GaDecoderDesc;
#define GA_DECODER_TENSOR_CORES 1
typedef struct GaDecoderLayout {
    int64_t gconv[3];
    int64_t w[7], b[7], gamma[7], beta[7];
    int64_t w8, b8, total;
    int32_t bn_channels, bn_offset[7];
} GaDecoderLayout;
/* Every buffer of the decoder workspace (device pointers; ga_decoder_views only computes addresses).  P = feat_res^2,
 * M = frames * S * S rows, frames 0 counted as 1.  Fp / dFp hold [frames][P,64] only when frames > 1 (4 floats otherwise). */
typedef struct GaDecoderViews {
    const float *F[4];              /* [P,64] NHWC: geo, conv1, conv2, conv3 (tensor-core path: F[0..2] TF32-rounded) */
    const float *wr;                /* [3][25*64*64] TF32-rounded conv weights (tensor-core path only) */
    const float *dF[2];             /* [P,64] ping-pong conv gradients */
    const float *Fp, *dFp;          /* [frames][P,64] stage-2 per-frame input maps and their gradients */
    const float *feat, *d_feat;     /* [M,72] [up-sampled features | u | v | 0 x 6] and its gradient */
    const float *Y[5], *Y6, *Y7;    /* [M,128] pre-BN outputs of layers 1-5; [M,384] of layers 6 and 7 (heads xyz, N, SH) */
    const float *dZa, *dZb;         /* [M,128] ping-pong pre-BN gradients of layers 5..1 */
    const float *dZ6, *dZ7;         /* [M,384] */
    const double *stat;             /* [4][1408]: sum, sumsq (forward), s1, s2 (backward) per BatchNorm channel */
    const float *coef;              /* [7][1408]: mean, rstd, a, b (forward), ga, m1, m2 (backward) */
} GaDecoderViews;
int ga_decoder_layout(const GaDecoderDesc *d, GaDecoderLayout *out);
size_t ga_decoder_workspace_bytes(const GaDecoderDesc *d);
/* pose_feat_nchw [frames,64,feat_res,feat_res] (NULL in stage 1): added to the geometry convs' output before the UV up-sampling
 * (pix_feature = pose_featmap + geom_featmap, model/network.py:58); d_pose_feat_nchw receives its gradient. */
int ga_decoder_forward(const GaDecoderDesc *d, const float *params, const float *geo_nchw, const float *pose_feat_nchw,
                       float *bn_running, void *workspace, float *dec_out, void *stream);
int ga_decoder_backward(const GaDecoderDesc *d, const float *params, void *workspace, const float *dec_out,
                        const float *d_dec_out, float *d_params, float *d_geo_nchw, float *d_pose_feat_nchw, void *stream);
int ga_decoder_views(const GaDecoderDesc *d, void *workspace, GaDecoderViews *out);
/* One decoder layer on the tensor cores (building block of ga_decoder_forward, exposed for unit tests):
 * Y[M,128] (+)= softplus(X * bn_a + bn_b)[M,K] W[128,K]^T + bias (bn_a == NULL: X used raw); optional per-column
 * sum / sum-of-squares accumulation (double[128]).  K % 8 == 0, K <= 128; ld* % 4 == 0. */
int ga_tc_linear_forward(int32_t M, int32_t K, const float *X, int32_t ldx, const float *bn_a, const float *bn_b, const float *W,
                         int32_t ldw, const float *bias, float *Y, int32_t ldy, int32_t accumulate, double *sum, double *sumsq,
                         void *stream);
/* The same for `heads` (1..3) layers that share X, in one launch: head h uses W + h w_hstride, writes Y + h y_hstride (floats) and
 * takes bias / sum / sumsq advanced by h v_hstride.  Each head's result is that of its own ga_tc_linear_forward. */
int ga_tc_linear_forward_heads(int32_t M, int32_t heads, int32_t K, const float *X, int32_t ldx, const float *bn_a, const float *bn_b,
                               const float *W, int32_t ldw, int64_t w_hstride, const float *bias, float *Y, int32_t ldy, int64_t y_hstride,
                               int32_t accumulate, double *sum, double *sumsq, int32_t v_hstride, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Fused image loss (utils/loss_utils.py:7-8,23-53 as combined at train.py:74-77):
 *   out3[0] = w_l1 * mean|image - gt| + w_ssim * (1 - ssim(image, gt)),  out3[1] = ssim, out3[2] = l1   (device floats)
 * image / gt [B,3,H,W].  The workspace (ga_loss_workspace_bytes) carries the SSIM partial-derivative maps from forward to
 * backward.  grad_out: device scalar dL/d out3[0] (NULL = 1).  d_image is overwritten.
 * ---------------------------------------------------------------------------------------------------------------- */
size_t ga_loss_workspace_bytes(int32_t B, int32_t H, int32_t W);
int ga_loss_forward(int32_t B, int32_t H, int32_t W, const float *image, const float *gt, float w_l1, float w_ssim,
                    void *workspace, float *out3, void *stream);
int ga_loss_backward(int32_t B, int32_t H, int32_t W, const float *image, const float *gt, float w_l1, float w_ssim,
                     const float *grad_out, void *workspace, float *d_image, void *stream);

/* Masked L1 depth loss on the mean depth of ga_rasterb_forward_depth(_train): depth [B,2,H,W] (plane 0 the mean m, plane 1 the
 * median), target [B,H,W] metric view-space z in the same world units (0 = no measurement).  A pixel counts when target > 0 and
 * plane 1 is non-zero (exactly where 1 - T_final >= 0.5, so 1 / A <= 2); N = the counted pixels of all B frames.
 *   out2[0] = lam / N * sum |m - target| over counted pixels (0 when N = 0),  out2[1] = N   (device floats)
 * N stays on the device and every sum has a fixed order (no atomics), so replays give the same loss bit for bit.  The backward
 * writes d_depth [B,H,W] = g lam sign(m - target) / N on counted pixels (sign(0) = 0) and 0 elsewhere, g = *grad_out (NULL = 1),
 * reading N from the workspace (ga_depth_loss_workspace_bytes) the forward of the same inputs filled.  Undersized workspaces and
 * NULL pointers are refused before any launch. */
size_t ga_depth_loss_workspace_bytes(int32_t B, int32_t H, int32_t W);
int ga_depth_loss_forward(int32_t B, int32_t H, int32_t W, const float *depth, const float *target, float lam, void *workspace,
                          size_t workspace_bytes, float *out2, void *stream);
int ga_depth_loss_backward(int32_t B, int32_t H, int32_t W, const float *depth, const float *target, const float *grad_out,
                           void *workspace, size_t workspace_bytes, float *d_depth, void *stream);

/* torch.optim.Adam step (amsgrad=False, weight_decay=0; model/avatar_model.py:148-155,264-267) on one contiguous buffer.
 * `step` is the 1-based count of this update; grad_scale multiplies the gradient first (1/world_size after an
 * all-reduce(sum)).  skip_flag (device int32, may be NULL): if non-zero when the kernel runs, nothing is updated — wired to the
 * batched rasterizer's overflow word so that a step rendered with an overflowed binning buffer is never committed. */
int ga_adam_step(int64_t n, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float lr, float beta1,
                 float beta2, float eps, int64_t step, float grad_scale, const int32_t *skip_flag, void *stream);
/* The same update with its scalars in DEVICE memory, hyper7 = [lr, beta1, beta2, eps, 1-beta1^step, sqrt(1-beta2^step),
 * grad_scale], so that a CUDA graph holding this launch follows the lr schedule / step count without re-capture. */
int ga_adam_step_dev(int64_t n, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, const float *hyper7,
                     const int32_t *skip_flag, void *stream);

/* Fused backward of one hidden decoder layer on the tensor cores (building block of ga_decoder_backward, exposed for unit
 * tests): from dZ_l / Y_l (BatchNorm backward applied on load with bwd_coef = [ga, m1, m2, mu, rstd] x 128, NULL: dY = dZ)
 * and Y_{l-1} (x = softplus(a y + b), prev_coef = [a, b, mu, rstd] x 128):  dW[128,128] += dY^T x  and
 * dZprev = (dY W) * sigmoid(z_{l-1}) with per-channel sums s1 = sum dZprev, s2 = sum dZprev * xhat_{l-1} (double[128]).
 * mode 0: as described; 1: store raw dY W; 2: dZprev += raw; 3: dZprev = (dZprev + dY W) * sigmoid, with statistics. */
int ga_tc_linear_backward(int32_t M, const float *dZ, const float *Y, int32_t ldg, const float *bwd_coef, const float *Yprev, int32_t ldp,
                          const float *prev_coef, const float *W, int32_t ldw, float *dW, int32_t lddw, float *dZprev, int32_t ldo,
                          int32_t mode, double *s1, double *s2, void *stream);
/* The same with the input width and form as arguments (ga_tc_linear_backward is kin = 128, x_raw = 0): only the first kin input
 * channels exist (kin % 4 == 0, kin <= 128; modes 0 and 3 need kin == 128): W and dW columns, Y_{l-1} and dZprev channels.
 * x_raw != 0 (modes 1, 2 only): x = Y_{l-1} as is (the network input), and prev_coef may be NULL. */
int ga_tc_linear_backward_ex(int32_t M, const float *dZ, const float *Y, int32_t ldg, const float *bwd_coef, const float *Yprev, int32_t ldp,
                             const float *prev_coef, const float *W, int32_t ldw, float *dW, int32_t lddw, float *dZprev, int32_t ldo,
                             int32_t mode, double *s1, double *s2, int32_t kin, int32_t x_raw, void *stream);

/* One 5x5, 64->64 channel, padding-2 convolution of the geometry net (model/modules.py:122-137; network.py:26,57) on the
 * tensor cores (building block of ga_decoder_forward/backward, exposed for unit tests).  Feature maps are NHWC [Hf*Hf][64],
 * weights [25 taps][64 ci][64 co]; operands must already hold TF32-representable values (ga_round_tf32).
 * mode 0: out = conv(in, w); mode 1: out = data gradient for in = dL/dY; mode 2: out (dW, same layout as w) += weight gradient
 * for in = X and w = dL/dY.  round_out != 0 rounds the result to TF32 (modes 0, 1). */
int ga_tc_conv5x5(int32_t mode, int32_t Hf, const float *in, const float *w, float *out, int32_t round_out, void *stream);
/* out[i] = in[i] rounded to TF32 (nearest, ties away; low 13 mantissa bits cleared).  n % 4 == 0; in-place allowed. */
int ga_round_tf32(const float *in, float *out, int64_t n, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * LPIPS perceptual distance, lpips.LPIPS(net='alex', version='0.1') in eval mode (train.py:89-91), forward and the gradient
 * with respect to in0.  Images planar fp32 [B,3,H,W], H, W >= 31; the network sees in * in_scale + in_shift (lpips's range
 * [-1,1]: 1, 0; images in [0,1]: 2, -1) through its scaling layer.  out[B] (device) = the distance per image pair.
 * Convolutions run TF32 with fp32 accumulation; nothing uses atomics, so both calls are bit-reproducible.
 *
 * weights: ga_lpips_weights_floats() device floats, 16-byte aligned, in this order (each block contiguous, row-major):
 *   for l = 1..5:  W_l  [C_out][tap][C_in]  (tap = ky * k + kx; conv1: [64][384] with index tap * 3 + c, zero from 363 on)
 *                  b_l  [C_out]
 *   for l = 2..5:  Wd_l [C_in][tap'][C_out] with tap' = (k-1-ky) * k + (k-1-kx)   (data gradient: flipped, transposed)
 *   for l = 1..5:  lin_l [C_out]   (the lin layers' 1x1 weights)
 *   with (C_in, C_out, k) = (3, 64, 11), (64, 192, 5), (192, 384, 3), (384, 256, 3), (256, 256, 3).
 * workspace: ga_lpips_workspace_bytes(B, H, W) bytes, 256-byte aligned; a forward leaves in it what its backward reads.
 * g[B] (device): dL/d out.  d_in0 [B,3,H,W] is overwritten.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct GaLpipsViews {
    float *relu[5];          /* relu_k maps NHWC [2B][H_k][W_k][C_k]: images 0..B-1 from in0, B..2B-1 from in1 */
    float *pool[2];          /* max-pool outputs NHWC [2B][..][..][C] (before conv2, conv3) */
    uint8_t *pool_arg[2];    /* window index 0..8 each pool output took */
    float *partials;         /* [5][B][128] per-CTA distance sums */
    float *in_scale;         /* in_scale of the last forward */
    float *dz[5];            /* backward: gradient at conv_k's output (before ReLU), NHWC [B][H_k][W_k][C_k] */
    float *dnext[4];         /* gradient reaching relu_k from slice k+1 (conv_{k+1} data gradient, un-pooled for k < 2) */
    float *dpool[2];         /* data gradients of conv2, conv3 at the pool outputs */
} GaLpipsViews;
size_t ga_lpips_weights_floats(void);
size_t ga_lpips_workspace_bytes(int32_t B, int32_t H, int32_t W);
int ga_lpips_forward(int32_t B, int32_t H, int32_t W, const float *weights, const float *in0, const float *in1, float in_scale,
                     float in_shift, void *workspace, float *out, void *stream);
int ga_lpips_backward(int32_t B, int32_t H, int32_t W, const float *weights, void *workspace, const float *g, float *d_in0, void *stream);
/* The workspace regions above (for tests and inspection). */
int ga_lpips_views(int32_t B, int32_t H, int32_t W, void *workspace, GaLpipsViews *out);

/* ------------------------------------------------------------------------------------------------------------------
 * Evaluation metrics, the sums behind torchmetrics' StructuralSimilarityIndexMeasure(data_range=dr) and
 * PeakSignalNoiseRatio(data_range=dr) as eval.py:20-35 uses them.  pred / target planar fp32 [B,C,H,W], H, W >= 11.
 *   ssim_sum[b] (device double) = sum over c and the cropped pixels 5 <= y < H-5, 5 <= x < W-5 of the SSIM map
 *     ((2 mx my + c1)(2 sxy + c2)) / ((mx^2 + my^2 + c1)(sx2 + sy2 + c2)),  c1 = (0.01 dr)^2, c2 = (0.03 dr)^2,
 *     moments under the 11x11 Gaussian window (sigma 1.5, taps built in fp32 as torch builds them) over the reflect-padded
 *     images, sx2 = max(E[x^2] - mx^2, 0), sy2 likewise, sxy = E[xy] - mx my; the image's SSIM is ssim_sum[b] / (C (H-10) (W-10)).
 *   sse[b] (device double) = sum over the whole image of (pred - target)^2.
 * Moments and sums in fp64; nothing uses atomics, so both outputs are bit-reproducible and do not depend on B.
 * partials: ga_metrics_partials_bytes(B, C, H, W) bytes, 8-byte aligned, scratch of the call (fp64 per-CTA sums).
 * ---------------------------------------------------------------------------------------------------------------- */
size_t ga_metrics_partials_bytes(int32_t B, int32_t C, int32_t H, int32_t W);
int ga_metrics_ssim_sse(int32_t B, int32_t C, int32_t H, int32_t W, const float *pred, const float *target, float data_range,
                        void *partials, double *ssim_sum, double *sse, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Screen-space mesh render (the posed-body overlay): B <= 8 frames of verts [B,V,3] (fp32), faces [F,3] (int32, each in
 * [0, V)), cams [B,40] (the ga_rasterb_* camera block: transposed view 0..15, transposed full projection 16..31).
 * adj_offsets [V+1] / adj_faces [3F]: vertex -> face CSR, faces of vertex v at adj_faces[adj_offsets[v] .. adj_offsets[v+1]),
 * each face once per corner it has there, in ascending face order (the normal is the normalised sum of their cross products).
 * Coverage: pixel centres, the Gaussian preprocess's projection and pixel convention, window coordinates snapped to 1/256
 * pixel, exact int64 edge functions with posmap.cu's tie rule; nearest face wins (perspective-correct depth, fp64, rounded
 * to fp32 once), lower face index at equal depth; no culling; a face with a corner at view depth <= 0.01 or beyond 2^20
 * pixels is not drawn.  Shading: glTF metallic-roughness BRDF (metallic 0.2, roughness 0.6, base colour base_*), one
 * headlight of intensity 3 along the camera's optical axis, no ambient, clamped to [0,1].
 * Outputs (every element written): face_id [B,H,W] (-1: nothing drawn), depth [B,H,W] (view-space z, 0: nothing drawn),
 * rgb [B,3,H,W] (background [B,3,H,W] where nothing is drawn, 0 if background is NULL).
 * workspace: ga_mesh_render_workspace_bytes(B, V, F, H, W) bytes, 256-byte aligned.  No floating-point atomics and no host
 * read-back: the outputs are bit-reproducible and a frame's do not depend on the batch it is drawn in.  H, W in [1, 16384].
 * ---------------------------------------------------------------------------------------------------------------- */
size_t ga_mesh_render_workspace_bytes(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W);
int ga_mesh_render(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, const float *verts, const int32_t *faces,
                   const int32_t *adj_offsets, const int32_t *adj_faces, const float *cams, float base_r, float base_g, float base_b,
                   const float *background, void *workspace, int32_t *face_id, float *depth, float *rgb, void *stream);
/* ga_mesh_shade_unlit: the unlit colour of the frames ga_mesh_render drew, from its face_id [B,H,W] and the same verts, faces, cams,
 * B in [1, 8].  At each pixel centre the drawn face's perspective-correct weights w_i = (E_i / area / z_i) / sum_k (E_k / area / z_k)
 * are recomputed in fp64 from the same snapped corners, then either
 *   colors [V,3] != NULL: rgb = sum_i w_i colors[v_i], or
 *   uvs [V,2] and texture [Th,Tw,3] (fp32, row 0 first, Th, Tw in [1, 16384]) != NULL: (s, t) = sum_i w_i uvs[v_i] in glTF's
 *   convention, x = s Tw - 0.5, y = t Th - 0.5 (texel (c, r) centred at (c, r)), and the bilinear blend of the four texels around
 *   (x, y), indices clamped to the edge.  The texels are blended as stored (display-encoded values, as a glTF viewer that does not
 *   decode sRGB to linear before filtering would; the unlit preview compares those values with the avatar's rendered ones).
 * All fp64 steps explicitly rounded, rgb [B,3,H,W] rounded to fp32 once; background [B,3,H,W] (0 if NULL) where face_id is -1 (or
 * not a face below F).  Exactly one of colors and (uvs, texture) is given.  Every element written, no atomics: bit-reproducible, and
 * a frame's output does not depend on the batch it is in. */
int ga_mesh_shade_unlit(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, const float *verts, const int32_t *faces, const float *cams,
                        const int32_t *face_id, const float *colors, const float *uvs, const float *texture, int32_t Th, int32_t Tw,
                        const float *background, float *rgb, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Animation player.
 * ga_motion_sample: a clip of T keys of J-joint axis-angle poses key_pose [T,J*3] (J = 24 for SMPL, 55 for SMPL-X's 165-wide
 * layout) and translations key_trans [T,3] (fp32, device), sampled at n fractional key indices times [n] (device double).
 * tau = clamp(times[k], 0, T-1) (NaN -> 0), i = floor(tau), f = tau - i.  Per joint, keys i and i+1 become unit quaternions,
 * the second negated when their dot product is negative, then slerp at f (normalised lerp above a dot of 1 - 1e-12); back to
 * axis-angle with w >= 0, so the angle is in [0, pi].  align [12] (device double): a row-major rotation R_a and an offset c;
 * the root becomes R_a R_root and the translation R_a lerp(t_i, t_i+1, f) + c.  All maths in fp64, rounded to fp32 once;
 * every element of pose_out [n,J*3] and trans_out [n,3] is written.  T >= 1, n >= 1.
 * ga_frame_pack: rendered frames image [B,3,H,W] (fp32, the batched rasterizer's C + T bg) -> interleaved bytes out
 * [B,H,W,channels].  q(x) = (uint8) clamp(fp32(fp32(x 255) + 0.5), 0, 255), NaN -> 0 (torchvision's save_image).
 * channels 3: q(image); final_T and bg may be NULL.  channels 4 (straight alpha; out 4-byte aligned): a = 1 - T with T =
 * final_T [B,H,W] (the rasterizer's image buffer, ga_raster_views), A = q(a); A = 0 gives (0,0,0,0), otherwise the colour
 * bytes are q((x - T bg_c) / a) and the fourth byte A.  Explicit fp32 roundings in that order (no contraction).
 * B in [1, 8]; H, W in [1, 16384].  No host read-back; both run on `stream` and are capturable in a CUDA graph.
 * ---------------------------------------------------------------------------------------------------------------- */
int ga_motion_sample(int32_t T, int32_t J, const float *key_pose, const float *key_trans, int32_t n, const double *times,
                     const double *align, float *pose_out, float *trans_out, void *stream);
int ga_frame_pack(int32_t B, int32_t H, int32_t W, int32_t channels, const float *image, const float *final_T, const float *bg,
                  uint8_t *out, void *stream);
/* ga_matte_pack: out[i] = q(mattes[i]) for n >= 1 values (ga_frame_pack's q; the mattes of ga_rasterb_forward_mattes as bytes). */
int ga_matte_pack(int64_t n, const float *mattes, uint8_t *out, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Soft silhouette (pose refinement against masks).  B in [1, 8] frames of verts [B,V,3] (fp32), faces [F,3] (int32, each in
 * [0, V)), cams [B,40] (the ga_rasterb_* camera block), H, W in [1, 16384], sigma > 0 in pixels^2.  Vertices are projected as
 * ga_mesh_render projects them, in fp32, not snapped; pixel (c, r) is centred at (c, r).  For face f and pixel centre p, d_f the
 * distance from p to the projected triangle: D_f = sigmoid(+-d_f^2 / sigma) (+ inside, - outside), 0 outside beyond
 * d_f^2 > sigma ln(1/1e-4 - 1); S = 1 - prod_f (1 - D_f).  A face with a corner at view depth <= 0.01 or beyond the 2^20-pixel
 * guard band, or with zero projected area, contributes nothing; no culling.
 * ga_silhouette_forward: sil [B,H,W]; with mask_u8 [B,H,W] (subject where the byte is >= 128) also loss [B] = mean_p (S - M)^2.
 *   mask_u8 may be NULL (then loss is not written and may be NULL).
 * ga_silhouette_backward: from the same inputs, mask_u8 required, and per-frame weights w [B] (device): d_verts [B,V,3] of
 *   sum_b w_b loss_b, through the projection, ready for ga_smpl(x)_vertices_backward.  adj_offsets [V+1] / adj_faces [3F]: the
 *   vertex -> face CSR of ga_mesh_render.
 * workspace: ga_silhouette_workspace_bytes(B, V, F, H, W) bytes, 256-byte aligned, sized by the shapes alone (no capacity).
 * Every output element is written.  No floating-point atomics and no host read-back: the outputs are bit-reproducible and a
 * frame's do not depend on the batch it is in.
 * ---------------------------------------------------------------------------------------------------------------- */
size_t ga_silhouette_workspace_bytes(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W);
int ga_silhouette_forward(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, float sigma, const float *verts, const int32_t *faces,
                          const float *cams, const uint8_t *mask_u8, void *workspace, float *sil, float *loss, void *stream);
int ga_silhouette_backward(int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, float sigma, const float *verts, const int32_t *faces,
                           const int32_t *adj_offsets, const int32_t *adj_faces, const float *cams, const uint8_t *mask_u8, const float *w,
                           void *workspace, float *d_verts, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Mesh extraction: truncated signed distance (TSDF) fusion of depth passes, then marching tetrahedra.  The grid holds samples at
 * origin + voxel (i, j, k), 0 <= i < nx etc., each side in [2, 512].  Its state is one caller buffer of ga_tsdf_state_bytes(d) =
 * 28 nx ny nz bytes: seven planes of nx ny nz 4-byte words, x fastest, in the order
 *   sdf (fp32, units of trunc, in [-1, 1]), weight (int32: views that observed the sample), carve (int32: views that saw no surface
 *   through it), r, g, b (fp32 sums of un-premultiplied colour), colour weight (int32).
 * ga_tsdf_reset zeroes the state (asynchronously, on `stream`).
 * ga_tsdf_integrate folds B in [1, 8] views into it, each sample's views in order (so the state does not depend on how views are
 *   split into calls): cams [B,40] (the ga_rasterb_* camera block), depth [B,2,H,W] (ga_rasterb_forward_depth; plane 1, the median,
 *   is read), image [B,3,H,W] rendered with bg = 0, final_T [B,H,W].  A sample is projected as the Gaussian preprocess projects a
 *   mean and reads the nearest pixel (pixel (c, r) centred at (c, r), ties to even); a view with view-space z <= 0.2 or the pixel
 *   outside the image is skipped.  With d the median depth there: d = 0 increments carve; else eta = d - z; eta < -trunc changes
 *   nothing; otherwise sdf <- (sdf weight + min(1, eta / trunc)) / (weight + 1), weight + 1, and where |eta| < trunc the colour sums
 *   gain image / (1 - final_T) and the colour weight 1.  No atomics: bit-reproducible.
 * ga_tsdf_mesh_count / ga_tsdf_mesh_emit: the zero level set by marching tetrahedra on the Kuhn split (each cube into the six
 *   tetrahedra (p, p + e_a, p + e_a + e_b, p + (1,1,1))).  A sample is outside (value +1) on the grid's outer layer or where
 *   carve >= min_carve (>= 1); otherwise inside (value -1) where weight = 0; otherwise inside iff sdf < 0 (value sdf).  count writes
 *   the vertex and face totals to totals [2] (device int32) and leaves offsets in the workspace (ga_tsdf_mesh_workspace_bytes(d));
 *   emit, with the same state, min_carve and workspace, writes verts [V,3] (the crossing of edge (p0, p1) at t = s0 / (s0 - s1)),
 *   colors [V,3] (the endpoints' mean colours interpolated at t; an endpoint without colour takes the other's, 0 if neither has one)
 *   and faces [F,3] int32 wound from inside to outside.  Vertices are ordered by owning sample p and slot (edges (p, p + d), d = x, y,
 *   z, xy, xz, yz, xyz), faces by cube, tetrahedron and triangle: the mesh is bit-reproducible, closed and 2-manifold.  emit writes no
 *   vertex at or past vertex_capacity and no face at or past face_capacity.
 * Bad sizes, NULL pointers, B outside [1, 8], a voxel or trunc that is not finite and > 0 are refused before anything launches.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct GaTsdfDesc {
    int32_t nx, ny, nz;          /* samples per axis, each in [2, 512]                                      */
    float origin[3];             /* world position of sample (0, 0, 0)                                      */
    float voxel;                 /* sample spacing, world units                                             */
    float trunc;                 /* truncation distance tau, world units                                    */
} GaTsdfDesc;
size_t ga_tsdf_state_bytes(const GaTsdfDesc *d);             /* 0 for a bad descriptor */
int ga_tsdf_reset(const GaTsdfDesc *d, void *state, void *stream);
int ga_tsdf_integrate(const GaTsdfDesc *d, int32_t B, int32_t H, int32_t W, const float *cams, const float *depth, const float *image,
                      const float *final_T, void *state, void *stream);
size_t ga_tsdf_mesh_workspace_bytes(const GaTsdfDesc *d);    /* 0 for a bad descriptor */
int ga_tsdf_mesh_count(const GaTsdfDesc *d, const void *state, int32_t min_carve, void *workspace, size_t workspace_bytes, int32_t *totals,
                       void *stream);
int ga_tsdf_mesh_emit(const GaTsdfDesc *d, const void *state, int32_t min_carve, const void *workspace, size_t workspace_bytes,
                      int64_t vertex_capacity, int64_t face_capacity, float *verts, float *colors, int32_t *faces, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Skin-weight transfer: per mesh vertex v of verts [V,3] (canonical space), the K joints it moves with, taken from the skinning rows
 * lbs [N,ld] of the N canonical Gaussian means [N,3] around it.
 *   Nearest means: the k nearest means by the fp32 squared distance d2 = __fadd_rn(__fadd_rn(dx dx, dy dy), dz dz), d = mean - v,
 *     each product and difference rounded on its own (no fused multiply-add); equal distances go to the lower Gaussian index.
 *   Blend (fp64, in neighbour order): c_i = 1 / (d2_i + eps^2), eps = 1e-3 world units; w_j = (sum_i c_i lbs_i[j]) / (sum_i c_i)
 *     for j < J (columns J..ld-1, e.g. SMPL-X's zero 56th, never count).
 *   Select: the K joints of largest positive w_j (equal weights go to the lower joint), renormalised to sum to 1 (the fp64 sum in
 *     slot order, each weight then rounded to fp32), written heaviest first as joints [V,K] uint8 and weights [V,K] fp32.  Slots left
 *     without a joint of positive weight are written (0, 0.0); a vertex whose blend is zero everywhere gets (0, 1.0) in slot 0.
 * One thread per vertex, no atomics: bit-reproducible.  Sizes outside 1 <= k <= min(16, N), 1 <= K <= min(8, J), 1 <= J <= ld <= 256,
 * V, N >= 1, and NULL pointers are refused before anything launches.
 * ---------------------------------------------------------------------------------------------------------------- */
int ga_skin_weights(int32_t V, int32_t N, int32_t J, int32_t ld, int32_t k, int32_t K, const float *verts, const float *means,
                    const float *lbs, uint8_t *joints, float *weights, void *stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Body-topology rig: the operators of its geometry fit and texture (rig.extract_body_rig).
 * ga_mesh_laplacian: y [V,3] = deg_v x_v - sum_{u in N(v)} x_u (the uniform graph Laplacian) for x [V,3] (fp32) and the vertex
 *   adjacency CSR offsets [V+1] / adj (neighbours of v at adj[offsets[v] .. offsets[v+1]), each in [0, V)).  In fp32: s = 0,
 *   s += x_u in stored order, y = fp32(deg x_v) - s, each step rounded on its own.  V in [1, 2^24].
 * ga_texture_pushpull: fills the texels of an S x S map, S in [1, 512], that mask [S,S] (uint8, nonzero: covered) leaves out, from
 *   the covered texels of image [C,S,S] (planar fp32, C in [1, 4]).  Down: level l+1 has side ceil(n_l / 2); its texel (r, c) gets
 *   weight w = sum of its children's weights (level 0: 1 per covered texel) and value (sum_k w_k v_k) / w over the children (2r + i,
 *   2c + j) with w_k > 0, in the order (0,0) (0,1) (1,0) (1,1), each product and sum rounded on its own (0 when w = 0); down to 1 x 1.
 *   Up: a texel of weight 0 takes its parent's (r / 2, c / 2) value, coarsest level first.  out [C,S,S]: covered texels copied from
 *   image bit for bit (uncovered texels of image are not read).  Every filled value is a convex combination of covered ones (0 when
 *   nothing is covered).  workspace: ga_texture_pushpull_workspace_bytes(S, C) bytes (0 for S = 1; 0 also for bad sizes), 256-byte
 *   aligned.
 * No atomics and no host read-back: bit-reproducible.  Bad sizes and NULL pointers are refused before anything launches.
 * ---------------------------------------------------------------------------------------------------------------- */
int ga_mesh_laplacian(int32_t V, const int32_t *offsets, const int32_t *adj, const float *x, float *y, void *stream);
size_t ga_texture_pushpull_workspace_bytes(int32_t S, int32_t C);
int ga_texture_pushpull(int32_t S, int32_t C, const float *image, const uint8_t *mask, void *workspace, size_t workspace_bytes, float *out,
                        void *stream);

#ifdef __cplusplus
}
#endif
#endif /* GAVATAR_H_ */
