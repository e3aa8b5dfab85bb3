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
typedef struct GaRasterSettings {
    int32_t P, H, W;
    float tanfovx, tanfovy, scale_modifier;
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
 * tanfovx 32, tanfovy 33.  `capacity` = number of (Gaussian, tile) instances the caller sized `binning` for; if a step needs
 * more, status[1] is set, the tiles that do not fit are rendered as empty and nothing is overrun — the caller re-runs with a
 * larger buffer (status[0] = the count needed).  status (device, 16 x int32, inside `img`): [0] instances, [1] overflow,
 * [2] backward segments, [4+b] first instance of frame b, [4+B] = [0]. */
typedef struct GaRasterBatchDesc {
    int32_t B, P, H, W;
    int64_t capacity;
    int64_t rot_stride, opac_stride;   /* floats between two frames' rotations / opacities: 4P / P, or 0 = shared */
    float scale_modifier;
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
int ga_rasterb_backward(const GaRasterBatchDesc *d, const float *cams, const float *bg, const float *means3D,
                        const float *colors, const float *scales, const float *rotations, const int32_t *radii,
                        const void *geom, const void *img, const void *binning, const float *dL_dout, void *scratch,
                        float *d_means3D, float *d_colors, float *d_scales, float *d_rotations, float *d_opacities,
                        float *d_means2D, void *stream);

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
int ga_posmap_layout(int32_t F, int32_t S, const float *uv_corners, int32_t *face_id, float *bary, void *stream);
int ga_posmap_fill(int32_t B, int32_t S, int32_t V, const float *verts, const int32_t *faces, const int32_t *face_id,
                   const float *bary, float *out, void *stream);

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
typedef struct GaDecoderViews {
    const float *conv3_nhwc, *feat, *y1, *y5, *bn_mean, *bn_rstd, *d_feat;
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

#ifdef __cplusplus
}
#endif
#endif /* GAVATAR_H_ */
