/*
 * gf_b200.h — C ABI of the H100-native (sm_90a) GaussianFormer hot path.
 *
 * Plain pointers and sizes only (no torch types).  Every pointer is a DEVICE pointer unless it
 * says "host".  Every entry point is asynchronous on the given stream and returns a GF_* status;
 * gf_last_error() gives the message for the calling thread.  The library never allocates or
 * frees device memory: scratch is a caller-provided workspace whose size comes from the matching
 * *_workspace_bytes() query (the reference instead grows torch byte tensors through
 * std::function callbacks — model/head/localagg/local_aggregate.cu:27-33,58-63).
 *
 * What each entry point replaces in the reference (paths relative to the reference tree):
 *
 *   gf_splat_forward   LocalAggregator::Aggregator::forward
 *                        model/head/localagg/src/aggregator.h:24-41, src/aggregator_impl.cu:152-252
 *                        model/head/localagg_prob/src/aggregator.h (variant = GF_SPLAT_PROB)
 *                        model/head/localagg_prob_fast/src/auxiliary.h:8-20 (radii_axes = 3)
 *                      plus, when the *_int / radii pointers are NULL, the host preparation of
 *                        model/head/localagg/local_aggregate/__init__.py:137-143
 *   gf_splat_backward  LocalAggregator::Aggregator::backward
 *                        model/head/localagg/src/aggregator.h:43-61, src/aggregator_impl.cu:256-307
 *                        model/head/localagg_prob/src/backward.cu:24-123 (variant = GF_SPLAT_PROB)
 *   gf_daf_forward     deformable_aggregation()
 *                        model/encoder/gaussian_encoder/ops/src/deformable_aggregation.cpp:4-18
 *                        .../ops/src/deformable_aggregation_cuda.cu:262-284
 *   gf_daf_backward    deformable_aggregation_grad()
 *                        .../ops/src/deformable_aggregation.cpp:20-38, ..._cuda.cu:287-313
 *
 *   gf_daf_fused_*     no native counterpart in the reference: the op call above together with the PyTorch code
 *                      around it in DeformableFeatureAggregation.forward
 *                        model/encoder/gaussian_encoder/deformable_module.py:213-228 (masked joint softmax of
 *                        the weights) and :242 (sum over the key points) -- an opt-in entry point (SURVEY.md 8f-2)
 *
 * The ABI is a superset of those boundaries: explicit stream, explicit class count C (the
 * reference hard-codes NUM_CHANNELS 18, model/head/localagg/src/config.h:15), 64-bit safe sizes,
 * caller-owned workspace and an int status.
 */
#ifndef GF_B200_H_
#define GF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GF_ABI_VERSION 2

/* status codes */
#define GF_OK 0
#define GF_ERR_INVALID_ARG 1   /* bad shape / NULL pointer / unsupported combination */
#define GF_ERR_WORKSPACE 2     /* workspace NULL, misaligned or smaller than *_workspace_bytes() */
#define GF_ERR_CUDA 3          /* a CUDA runtime call failed (message has cudaGetErrorString) */
#define GF_ERR_UNSUPPORTED 4   /* e.g. class count outside the compiled range */

/* element type of the deformable-aggregation feature table and maps (the feat_dtype of the gf_daf_*_ex entry points) */
#define GF_DTYPE_F32 0
#define GF_DTYPE_F16 1         /* IEEE binary16 (__half, torch.float16) */
#define GF_DTYPE_BF16 2        /* bfloat16 (__nv_bfloat16, torch.bfloat16) */

/* splat variants */
#define GF_SPLAT_BASE 0        /* local_aggregate:            logits                       */
#define GF_SPLAT_PROB 1        /* local_aggregate_prob(_fast): logits, bin_logits, density  */

/* bits of the device-side status word (gf_splat_read_flags) — the conditions the reference's
 * Python wrapper asserts on (local_aggregate/__init__.py:138,140,142) */
#define GF_FLAG_POINT_OUT_OF_GRID 1u
#define GF_FLAG_MEAN_OUT_OF_GRID 2u
#define GF_FLAG_RADIUS_LT_1 4u
#define GF_FLAG_GENERIC_PATH 256u /* informational: points were not in canonical voxel order */

typedef void *gf_stream_t; /* a cudaStream_t (NULL = legacy default stream) */

typedef struct gf_splat_desc {
    int32_t G;          /* Gaussians (P in the reference) */
    int32_t N;          /* query points */
    int32_t C;          /* classes / channels (18 for nuScenes-SurroundOcc) */
    int32_t H, W, D;    /* voxel grid */
    int32_t variant;    /* GF_SPLAT_BASE | GF_SPLAT_PROB */
    int32_t radii_axes; /* 1: one radius per Gaussian, 3: per-axis radii (prob_fast) */
    int32_t cov_stride; /* floats per Gaussian in `cov`: 6 = (xx,yy,zz,xy,yz,xz); 9 = row-major
                           3x3 from which entries [0,4,8,1,5,2] are taken (__init__.py:143) */
    /* host-preparation parameters, used when points_int / means_int / radii are NULL */
    float pc_min[3];
    float grid_size;
    float scale_multiplier;
    int32_t radii_min;  /* <=0: no clamp (base variant); >=1: radii.clamp(min) (prob variants) */
    /* ---- ABI 2: explicit batch (the reference op is per sample, local_aggregate/__init__.py:128; SURVEY.md 8b/8e) ---- */
    int32_t batch;      /* samples per call, B >= 1 (0 is read as 1).  Every input / output / gradient tensor carries a
                           leading dimension B with dense strides ([B,N,3], [B,G,3], [B,G], [B,G,C], [B,N,C], ...); all B
                           samples are processed by ONE grid per kernel, and the workspace is B times the B = 1 size */
    int32_t pts_shared; /* != 0: pts / points_int are ONE [N,3] array shared by every sample of the batch (the voxel
                           centres of the occupancy grid, dataset/transform_3d.py:487-499) instead of [B,N,3] */
} gf_splat_desc;

/* Inputs of both passes.  points_int / means_int / radii mirror the reference's native
 * boundary; pass NULL to have them derived on the device from pts / means / scales exactly as
 * the reference's Python wrapper does (fp32 subtract, fp32 divide, truncate; ceil for radii). */
typedef struct gf_splat_inputs {
    const float *pts;         /* [N,3] */
    const int32_t *points_int;/* [N,3] or NULL */
    const float *means;       /* [G,3] */
    const int32_t *means_int; /* [G,3] or NULL */
    const float *opacities;   /* [G] */
    const float *semantics;   /* [G,C] */
    const float *cov;         /* [G,cov_stride] inverse covariance */
    const int32_t *radii;     /* [G] or [G,3], or NULL */
    const float *scales;      /* [G,3]; read when radii == NULL or cov == NULL */
    /* ---- ABI 2: head pre-op fusion (SURVEY.md 8f-1) ---- */
    const float *rotations;   /* [G,4] quaternions (w,x,y,z), any norm > 0, or NULL.  With cov == NULL the inverse
                                 covariance is built on the device as R^T diag(1/s^2) R from scales and rotations -- the
                                 closed form of GaussianHead.prepare_gaussian_args' Cov = (S R)^T (S R),
                                 Cov.cpu().inverse().cuda() (model/head/gaussian_head.py:111-119; quaternion -> matrix
                                 as model/utils/utils.py:20-66) -- inside the pack kernel */
} gf_splat_inputs;

typedef struct gf_splat_outputs {
    float *logits;      /* [N,C]; may be NULL when logits_cn, argmax or ce_partials is requested instead */
    float *bin_logits;  /* [N]  (prob only) */
    float *density;     /* [N]  (prob only) */
    float *probability; /* [N]  (prob only; saved for backward like the reference) */
    uint8_t *argmax;    /* [N]  optional, NULL = off: class with the largest logit per point (lowest
                           index on ties) — the `argmax(dim=1)` of GaussianHead.forward
                           (model/head/gaussian_head.py:185) fused into the render epilogue */
    /* ---- ABI 2: post-op fusion toward the loss (SURVEY.md 8f-3); all optional, NULL = off ---- */
    float *logits_cn;   /* [C,N] per sample: the logits class-major, i.e. the `semantics[None].transpose(1, 2)` /
                           `[1, C, N]` layout GaussianHead hands to the loss (gaussian_head.py:165-175), written by the
                           render epilogue; `logits` may then be NULL (inference: the [N,C] copy never exists) */
    const uint8_t *labels;      /* [N] per sample: target class per point, 255 = ignore (loss/occupancy_loss.py:113-127) */
    const float *class_weights; /* [C] (shared by the batch) or NULL = all ones */
    float *ce_partials; /* [gf_splat_ce_partials(desc), 2] fully overwritten: per render CTA (sum_n w[y_n] * nll_n,
                           sum_n w[y_n]) of CE_ssc_loss = nn.CrossEntropyLoss(weight, ignore_index=255, 'mean')
                           (loss/occupancy_loss.py:164-178) over the CTA's points; loss = sum(col 0) / sum(col 1).
                           Needs labels; tile path only (N == H*W*D, canonical order) */
} gf_splat_outputs;

typedef struct gf_splat_grads {
    /* upstream */
    const float *logits_grad;     /* [N,C] */
    const float *bin_logits_grad; /* [N] (prob only) */
    const float *density_grad;    /* [N] (prob only) */
    /* saved forward outputs (prob only) */
    const float *logits;          /* [N,C] */
    const float *bin_logits;      /* [N] */
    const float *probability;     /* [N] */
    /* results: fully overwritten */
    float *means_grad;            /* [G,3] */
    float *opacity_grad;          /* [G] */
    float *semantics_grad;        /* [G,C] */
    float *cov_grad;              /* cov_stride 6: [G,6] in (xx,yy,zz,xy,yz,xz) order; cov_stride 9: [G,9] row-major
                                     3x3, entries [0,4,8,1,5,2] carry the gradient, [3,6,7] are written as 0.
                                     May be NULL when in->cov == NULL (scales + rotations input) */
    /* ---- ABI 2: gradients of the fused pre-op (in->cov == NULL, in->rotations != NULL); fully overwritten ---- */
    float *scales_grad;           /* [G,3] through Sigma^-1 only (the radii are detached, __init__.py:134) */
    float *rotations_grad;        /* [G,4] w.r.t. the un-normalised quaternion */
} gf_splat_grads;

typedef struct gf_daf_desc {
    int32_t batch;      /* B */
    int32_t num_cams;   /* M */
    int32_t num_feat;   /* F = sum_l h_l*w_l */
    int32_t num_embeds; /* C */
    int32_t num_scale;  /* L */
    int32_t num_pts;    /* P */
    int32_t num_groups; /* Gr, divides C */
} gf_daf_desc;

#define GF_DAF_MAX_LEVELS 8

/* feature_maps_format (ops/deformable_aggregation.py:78-117, forward direction): L maps
 * [B*M, C, h_l, w_l] (contiguous) <-> one channels-last table [B*M, F, C], F = sum_l h_l*w_l,
 * level l occupying rows [sum_{k<l} h_k*w_k, ...).  The reference builds it with reshape + cat +
 * permute and leaves the transposing copy to every later .contiguous(). */
typedef struct gf_daf_format_desc {
    int32_t batch_cams; /* B*M */
    int32_t num_embeds; /* C */
    int32_t num_scale;  /* L <= GF_DAF_MAX_LEVELS */
    int32_t hw[GF_DAF_MAX_LEVELS]; /* h_l*w_l */
} gf_daf_format_desc;

int gf_abi_version(void);
const char *gf_last_error(void);

/* number of classes the splat kernels were compiled for: returns how many values were written
 * to out[] (at most cap). */
int gf_splat_supported_classes(int32_t *out, int cap);

size_t gf_splat_forward_workspace_bytes(const gf_splat_desc *desc);
/* rows of out->ce_partials for this desc (render CTAs of the tile path x batch); 0 when the tile path does not apply */
int gf_splat_ce_partials(const gf_splat_desc *desc);
size_t gf_splat_backward_workspace_bytes(const gf_splat_desc *desc);

int gf_splat_forward(const gf_splat_desc *desc, const gf_splat_inputs *in,
                     const gf_splat_outputs *out, void *workspace, size_t workspace_bytes,
                     gf_stream_t stream);

int gf_splat_backward(const gf_splat_desc *desc, const gf_splat_inputs *in,
                      const gf_splat_grads *grads, void *workspace, size_t workspace_bytes,
                      gf_stream_t stream);

/* ---- backward flags: gf_splat_backward_workspace_bytes_ex / gf_splat_backward_ex are the two functions above with a
 * flags word; the functions above are these with flags 0.  Unknown bits: the query returns 0 and the backward
 * GF_ERR_INVALID_ARG, with a message, before any CUDA call.
 *
 * GF_BWD_DETERMINISTIC: bit-reproducible gradients.  Every gradient is a sum in an order fixed by the inputs alone
 * (no floating-point atomics), so repeated calls, a sample run alone or inside a batch, and GPUs with different SM
 * counts give identical bytes.  The workspace is larger (gf_splat_backward_workspace_bytes_ex with the same flags). */
#define GF_BWD_DETERMINISTIC 1u

size_t gf_splat_backward_workspace_bytes_ex(const gf_splat_desc *desc, uint32_t flags);

int gf_splat_backward_ex(const gf_splat_desc *desc, uint32_t flags, const gf_splat_inputs *in,
                         const gf_splat_grads *grads, void *workspace, size_t workspace_bytes,
                         gf_stream_t stream);

/* Copies the status word of the last gf_splat_forward that used `workspace` to *host_flags
 * (GF_FLAG_* bits) and synchronises the stream.  The reference raises AssertionError from Python
 * for the same conditions. */
int gf_splat_read_flags(const void *workspace, gf_stream_t stream, uint32_t *host_flags);

/* out[B,P,C] is fully overwritten. */
int gf_daf_forward(const gf_daf_desc *desc, const float *mc_ms_feat, const int32_t *spatial_shape,
                   const int32_t *scale_start_index, const float *sample_location,
                   const float *weights, float *output, gf_stream_t stream);

/* Accumulates (+=) into the three gradient buffers like the reference's atomics do; the caller
 * zero-fills them first (ops/deformable_aggregation.py:55-57). */
int gf_daf_backward(const gf_daf_desc *desc, const float *mc_ms_feat, const int32_t *spatial_shape,
                    const int32_t *scale_start_index, const float *sample_location,
                    const float *weights, const float *grad_output, float *grad_mc_ms_feat,
                    float *grad_sampling_location, float *grad_weights, gf_stream_t stream);

/* One pass over the data in either direction: inverse == 0 gathers the L maps into `table`
 * (fully overwritten); inverse != 0 scatters `table` back into the L maps (fully overwritten; this is the
 * gradient of the forward direction).  maps[l] are device pointers, the array itself lives on the host. */
int gf_daf_format(const gf_daf_format_desc *desc, float *const *maps, float *table, int inverse,
                  gf_stream_t stream);

/* ---- fused caller path of the deformable aggregation (opt-in; the entry points above stay the drop-in) ----
 *
 * For every anchor a (num_pts = A * pts_per_anchor sampling points per batch element, anchor-major) and
 * group g, with e running over the anchor's (key point k, camera m, level l) entries:
 *
 *   on_e   = point_mask[b,a,k,m] (or 1 if NULL)  &  weight_mask[b,a,k,m,l,g] (or 1 if NULL)
 *   w_e    = on_e ? exp(logit_e) / sum_{e' on} exp(logit_e') : 0        (all weights 0 when no entry is on)
 *   out[b,a,c] = sum_k gf_daf_forward(...)[b, a*K + k, c]  evaluated with the weights w
 *
 * which is deformable_module.py:213-228 + :242 (weights[~mask] = -inf; weights[all_miss] = 0; softmax over the
 * flattened (k, m, l) axis; * (1 - all_miss); DAF.apply; .sum(dim=2)).  Masks are bytes (0 / non-zero; a
 * torch.bool tensor).  `stats` [B, A, Gr, 2] receives (max * log2(e), 1 / sum) per anchor and group and is what
 * the backward needs besides the forward output.  Supported when gf_daf_fused_supported() != 0:
 * num_embeds % 128 == 0, groups a power of two that divides num_embeds / 4 into power-of-two runs,
 * num_cams * num_scale <= 32; other shapes return GF_ERR_UNSUPPORTED (use the unfused entry points). */
typedef struct gf_daf_fused_desc {
    gf_daf_desc d;
    int32_t pts_per_anchor; /* K; d.num_pts % K == 0 */
} gf_daf_fused_desc;

int gf_daf_fused_supported(const gf_daf_fused_desc *desc);

/* output [B, A, C] and stats [B, A, Gr, 2] are fully overwritten. */
int gf_daf_fused_forward(const gf_daf_fused_desc *desc, const float *mc_ms_feat, const int32_t *spatial_shape,
                         const int32_t *scale_start_index, const float *sample_location,
                         const float *weight_logits, const uint8_t *point_mask, const uint8_t *weight_mask,
                         float *output, float *stats, gf_stream_t stream);

/* grad_weight_logits [B, A, K, M, L, Gr] is fully overwritten; grad_mc_ms_feat and grad_sampling_location are
 * accumulated into (+=) like gf_daf_backward: the caller zero-fills them. */
int gf_daf_fused_backward(const gf_daf_fused_desc *desc, const float *mc_ms_feat, const int32_t *spatial_shape,
                          const int32_t *scale_start_index, const float *sample_location,
                          const float *weight_logits, const uint8_t *point_mask, const uint8_t *weight_mask,
                          const float *stats, const float *output, const float *grad_output,
                          float *grad_mc_ms_feat, float *grad_sampling_location, float *grad_weight_logits,
                          gf_stream_t stream);

/* ---- half-precision feature tables: the five deformable-aggregation entry points with the element type of the
 * feature table (and, for gf_daf_format_ex, of the maps) given as feat_dtype = GF_DTYPE_F32 | GF_DTYPE_F16 |
 * GF_DTYPE_BF16.  The entry points above are these with GF_DTYPE_F32.
 *
 * The kernels convert every table value to fp32 where they load it and then run the fp32 arithmetic, so outputs are
 * bit-identical to the GF_DTYPE_F32 call on the upcast table.  Everything except the table stays fp32, including
 * grad_mc_ms_feat: the backward accumulates (+=) into an fp32 [B, M, F, C] buffer the caller zero-fills, and the
 * caller rounds it to the table's type once, after the call.  gf_daf_format_ex moves data in feat_dtype both ways.
 * An unknown feat_dtype returns GF_ERR_INVALID_ARG before any CUDA call. */
int gf_daf_forward_ex(const gf_daf_desc *desc, int32_t feat_dtype, const void *mc_ms_feat,
                      const int32_t *spatial_shape, const int32_t *scale_start_index, const float *sample_location,
                      const float *weights, float *output, gf_stream_t stream);

int gf_daf_backward_ex(const gf_daf_desc *desc, int32_t feat_dtype, const void *mc_ms_feat,
                       const int32_t *spatial_shape, const int32_t *scale_start_index, const float *sample_location,
                       const float *weights, const float *grad_output, float *grad_mc_ms_feat,
                       float *grad_sampling_location, float *grad_weights, gf_stream_t stream);

int gf_daf_fused_forward_ex(const gf_daf_fused_desc *desc, int32_t feat_dtype, const void *mc_ms_feat,
                            const int32_t *spatial_shape, const int32_t *scale_start_index,
                            const float *sample_location, const float *weight_logits, const uint8_t *point_mask,
                            const uint8_t *weight_mask, float *output, float *stats, gf_stream_t stream);

int gf_daf_fused_backward_ex(const gf_daf_fused_desc *desc, int32_t feat_dtype, const void *mc_ms_feat,
                             const int32_t *spatial_shape, const int32_t *scale_start_index,
                             const float *sample_location, const float *weight_logits, const uint8_t *point_mask,
                             const uint8_t *weight_mask, const float *stats, const float *output,
                             const float *grad_output, float *grad_mc_ms_feat, float *grad_sampling_location,
                             float *grad_weight_logits, gf_stream_t stream);

int gf_daf_format_ex(const gf_daf_format_desc *desc, int32_t feat_dtype, void *const *maps, void *table, int inverse,
                     gf_stream_t stream);

/* ---- backward flags of the deformable aggregation: the two backward _ex entry points above with a flags word (the
 * GF_BWD_* bits of the splat backward) and a caller-provided workspace.  Flags 0: the _ex call itself; the query
 * returns 0 and the workspace may be NULL.  Unknown bits: the query returns 0 and the call GF_ERR_INVALID_ARG, with a
 * message, before any CUDA call.  A workspace smaller than the query (same desc and flags): GF_ERR_INVALID_ARG.
 *
 * GF_BWD_DETERMINISTIC: bit-reproducible gradients (repeated calls, a sample alone or inside a batch, any SM count).
 * The feature gradient is gathered per feature row instead of scattered with atomics: the visible (point, camera,
 * level) pairs are sorted by their bilinear cell, and every row sums its entries in a fixed order.  The weight (fused:
 * logit) and location gradients come from the default fast kernels with their feature atomics left out (those kernels
 * reduce them in a fixed order already) or, for the shapes of the general kernel, from a variant that sums them in a
 * fixed order.  The workspace is sized for every pair visible, in closed form from the desc (no device query); the route needs
 * B * P * M * L < 2^31 and B * M * (2 F + 2 L) < 2^31, otherwise the query returns 0 and the call GF_ERR_UNSUPPORTED,
 * with a message.  The += contract of the gradient buffers is unchanged. */
size_t gf_daf_backward_workspace_bytes(const gf_daf_desc *desc, uint32_t flags);

int gf_daf_backward_ex2(const gf_daf_desc *desc, int32_t feat_dtype, uint32_t flags, const void *mc_ms_feat,
                        const int32_t *spatial_shape, const int32_t *scale_start_index, const float *sample_location,
                        const float *weights, const float *grad_output, float *grad_mc_ms_feat,
                        float *grad_sampling_location, float *grad_weights, void *workspace, size_t workspace_bytes,
                        gf_stream_t stream);

size_t gf_daf_fused_backward_workspace_bytes(const gf_daf_fused_desc *desc, uint32_t flags);

int gf_daf_fused_backward_ex2(const gf_daf_fused_desc *desc, int32_t feat_dtype, uint32_t flags,
                              const void *mc_ms_feat, const int32_t *spatial_shape, const int32_t *scale_start_index,
                              const float *sample_location, const float *weight_logits, const uint8_t *point_mask,
                              const uint8_t *weight_mask, const float *stats, const float *output,
                              const float *grad_output, float *grad_mc_ms_feat, float *grad_sampling_location,
                              float *grad_weight_logits, void *workspace, size_t workspace_bytes, gf_stream_t stream);

/* ---- camera projection of 3-D key points: DeformableFeatureAggregation.project_points
 * (model/encoder/gaussian_encoder/deformable_module.py:287-305) in the layout the op takes (:207-209), the stage
 * between the key-point generator and gf_daf_fused_*.  For point p (anchor-major, p = a * K + k) of sample b and camera
 * m, with P = projection_mat[b, m] (row-major 4x4):
 *
 *   x, y, z  = P[0:3, :] . (X, Y, Z, 1)               in fp64 from the fp32 inputs
 *   zc       = max(z, (double)1e-5f)                  (a NaN depth stays NaN, as torch.clamp)
 *   u, v     = x / zc / W, y / zc / H                 in fp64; (W, H) = image_wh[b, m], no division when NULL
 *   loc[b, p, m]        = (float(u), float(v))         the only rounding
 *   point_mask[b, p, m] = z > (double)1e-5f && 0 < loc.x < 1 && 0 < loc.y < 1   (on the fp32 loc: the sampling
 *                                                      kernels' own camera gate)
 *
 * key_points [B, P, 3], projection_mat [B, M, 4, 4], image_wh [B, M, 2] or NULL, loc [B, P, M, 2] (8-byte aligned),
 * point_mask [B, P, M] bytes; loc and point_mask are fully overwritten.
 *
 * gf_daf_project_backward: grad_key_points [B, P, 3] is fully overwritten with the key-point gradient of loc given
 * grad_loc [B, P, M, 2] (8-byte aligned), summed in fp64 over the cameras the mask lets through, in ascending order,
 * and rounded once: g_u (P0j - u' P2j) / (z W) + g_v (P1j - v' P2j) / (z H) with u' = x / z, v' = y / z.  Masked
 * cameras contribute nothing whatever their grad_loc.  No gradient reaches projection_mat or image_wh.
 *
 * Both re-evaluate the same projection, need no workspace and do not synchronise.  Negative sizes, NULL pointers for
 * non-empty work and B * P * M >= 2^31 are refused before any CUDA call. */
int gf_daf_project(int32_t batch, int32_t num_pts, int32_t num_cams, const float *key_points,
                   const float *projection_mat, const float *image_wh, float *loc, uint8_t *point_mask,
                   gf_stream_t stream);

int gf_daf_project_backward(int32_t batch, int32_t num_pts, int32_t num_cams, const float *key_points,
                            const float *projection_mat, const float *image_wh, const float *grad_loc,
                            float *grad_key_points, gf_stream_t stream);

/* ---- key points of Gaussian anchors: SparseGaussian3DKeyPointsGenerator.forward
 * (model/encoder/gaussian_encoder/deformable_module.py:51-90), the stage in front of gf_daf_project.  For anchor row
 * x = anchor[b, a, :] (anchor_dim >= 10 columns: xyz logits, scale logits, quaternion (w, x, y, z), then anything) and
 * key point k (the num_fixed fixed points first, then the num_learnable learnable ones):
 *
 *   sig(v)  = 1 / (1 + exp(-clamp(v, -9.21f, 9.21f)))                                    safe_sigmoid
 *   xyz     = lo + extent * sig(x[0:3])
 *   gs      = scale_lo + scale_extent * sig(x[3:6])
 *   s_k     = fix_scale[k]                                                               k <  num_fixed
 *           = (sig(learnable_logits[b, a, k - num_fixed]) - 0.5) * learnable_fixed_scale   k >= num_fixed
 *   key_points[b, a, k] = R^T (s_k * gs) + xyz,   R = get_rotation_matrix(x[6:10]) (model/utils/utils.py:20-69,
 *                                                 F.normalize with epsilon (double)1e-12f first)
 *
 * in fp64 from the fp32 inputs, each output rounded to fp32 once.  The descriptor's floats are the fp32 values the
 * reference's fp32 tensors multiply by: lo = pc_range[0:3], extent = float(pc_range[3:6] - pc_range[0:3]),
 * scale_lo = scale_range[0], scale_extent = float(scale_range[1] - scale_range[0]).
 *
 * anchor [B, A, anchor_dim], fix_scale [num_fixed, 3], learnable_logits [B, A, num_learnable, 3] (the pre-sigmoid
 * learnable_fc output; NULL when num_learnable == 0), key_points [B, A, num_fixed + num_learnable, 3], fully
 * overwritten.
 *
 * gf_daf_anchor_key_points_backward: given grad_key_points [B, A, K, 3], fully overwrites grad_anchor
 * [B, A, anchor_dim] (columns 10 and up are 0) and grad_learnable [B, A, num_learnable, 3] (the gradient of the
 * pre-sigmoid logits; may be NULL when num_learnable == 0).  One thread per anchor sums over k in ascending order in
 * fp64 without atomics, so the gradients are bit-reproducible.  The clamps pass the gradient where
 * -9.21f <= v <= 9.21f, bounds included (torch.clamp's backward), and block it elsewhere.
 *
 * Both need no workspace and do not synchronise.  A NULL desc, negative sizes, anchor_dim < 10, no key points for
 * non-empty work and NULL pointers for non-empty work are GF_ERR_INVALID_ARG; B * A * K >= 2^31 or
 * B * A * anchor_dim >= 2^31 is GF_ERR_UNSUPPORTED; all before any CUDA call. */
typedef struct gf_daf_kps_desc {
    int32_t batch, num_anchors, anchor_dim, num_fixed, num_learnable;
    float lo[3], extent[3], scale_lo, scale_extent, learnable_fixed_scale;
} gf_daf_kps_desc;

int gf_daf_anchor_key_points(const gf_daf_kps_desc *desc, const float *anchor, const float *fix_scale,
                             const float *learnable_logits, float *key_points, gf_stream_t stream);

int gf_daf_anchor_key_points_backward(const gf_daf_kps_desc *desc, const float *anchor, const float *fix_scale,
                                      const float *learnable_logits, const float *grad_key_points,
                                      float *grad_anchor, float *grad_learnable, gf_stream_t stream);

/* ---- occupancy loss of one supervised layer: OccupancyLoss.loss_voxel (loss/occupancy_loss.py:102-149) as every
 * shipped config runs it, ce_weight * CE + lovasz_weight * Lovasz-softmax (loss/utils/lovasz_softmax.py:157-234),
 * with its gradient.  Inputs: pred [B, C, N] (logits, or probabilities with GF_OCC_PROBS) in one of two layouts,
 * labels [B, N] int64, mask [B, N] bytes or NULL (all voxels), class_weights [C].
 *
 *   S   = {(b, n) : mask, and label != empty_label when empty_label >= 0}, b-major, n ascending (one pool: B > 1 is
 *         the batch pooled, not averaged per sample)
 *   CE  = sum w[y] (-log p_y) / sum w[y] over the s in S with y != ignore_index; p = softmax_c(pred) (GF_OCC_LOGITS)
 *         or clamp(pred, 1e-6f, 1 - 1e-6f) (GF_OCC_PROBS).  NaN when no voxel counts, as PyTorch's mean
 *   V   = {s in S : y != lovasz_ignore} in S order; r = p (GF_OCC_LOGITS) or pred (GF_OCC_PROBS).  A label outside
 *         [0, C) stays in V as background of every class.  Class c is present if some s in V has y = c.  For each:
 *         e_s = |[y_s = c] - r_{s,c}| sorted descending, equal errors in ascending position in V (a stable sort);
 *         fg in that order, G = sum fg, I_k = G - sum_{j<=k} fg_j, U_k = G + sum_{j<=k} (1 - fg_j),
 *         J_k = 1 - I_k / U_k, Delta_k = J_k - J_{k-1} (J_{-1} = 0), L_c = sum_k e_(k) Delta_k.
 *         Lovasz = mean of L_c over the present classes, 0 when none is
 *   loss_out[3] = { weight * (ce_weight * CE + lovasz_weight * Lovasz), CE, Lovasz }, fully overwritten
 *
 * grad_out (NULL: loss only) receives d loss_out[0] / d pred in pred's layout, every entry written (0 outside S).  No
 * gradient flows through Delta, and |.| at 0 passes 0 (torch.abs).  The arithmetic is fp64 from the fp32 inputs; each
 * error is rounded to fp32 once to be sorted, and the loss and every gradient entry once at the end.  Every sum runs
 * in a fixed order without floating-point atomics, so loss and gradient are bit-reproducible from call to call.
 *
 * The workspace is sized from the desc for the worst case |V| = B * N (gf_occ_loss_workspace_bytes; 16 * C * B * N
 * bytes for the sort plus O(B * N) more), 256-byte aligned; the counts stay on the device, so the call never
 * synchronises and can be captured in a CUDA graph.  The first uint32 of the workspace is the call's status word:
 * GF_FLAG_LABEL_OUT_OF_RANGE when a label in S is outside [0, C) and neither ignore_index nor lovasz_ignore.
 *
 * Supported: C in gf_splat_supported_classes(), B * N * C < 2^31.  Otherwise, and for a NULL desc, unknown branch or
 * layout, NULL pointers or a small workspace, the call fails before any CUDA call. */
#define GF_OCC_LOGITS 0
#define GF_OCC_PROBS 1
#define GF_OCC_VOXEL_MAJOR 0   /* pred[b, c, n] at (b * N + n) * C + c: the transposed view of the splat's [B, N, C] */
#define GF_OCC_CLASS_MAJOR 1   /* pred[b, c, n] at (b * C + c) * N + n: the contiguous [B, C, N] of logits_cn */
#define GF_FLAG_LABEL_OUT_OF_RANGE 8u

typedef struct gf_occ_loss_desc {
    int32_t batch;         /* B */
    int32_t N;             /* voxels per sample */
    int32_t C;             /* classes */
    int32_t branch;        /* GF_OCC_LOGITS | GF_OCC_PROBS */
    int32_t layout;        /* GF_OCC_VOXEL_MAJOR | GF_OCC_CLASS_MAJOR, for pred and grad_out */
    int32_t ignore_index;  /* CE ignore label (255) */
    int32_t lovasz_ignore; /* label left out of V (17 in the shipped configs) */
    int32_t empty_label;   /* ignore_empty: voxels with this label leave S; < 0 = off */
    float weight, ce_weight, lovasz_weight;
} gf_occ_loss_desc;

size_t gf_occ_loss_workspace_bytes(const gf_occ_loss_desc *desc);

int gf_occ_loss(const gf_occ_loss_desc *desc, const float *pred, const int64_t *labels, const uint8_t *mask,
                const float *class_weights, float *loss_out, float *grad_out, void *workspace, size_t workspace_bytes,
                gf_stream_t stream);

/* ---- submanifold sparse convolution: spconv's SubMConv3d(c_in, c_out, k, stride 1, padding (k-1)/2) as the
 * encoder's SparseConv3D (model/encoder/gaussian_encoder/spconv3d_module.py:10-83) calls it, forward and backward.
 * Inputs: features [N, c_in] fp32, indices [N, 4] int32 rows (b, x, y, z) in any order, weight in spconv 2.x layout
 * [c_out, k, k, k, c_in], bias [c_out] or NULL.
 *
 *   valid row   0 <= b < batch and (x, y, z) inside [0, X) x [0, Y) x [0, Z)
 *   voxel       occupied when it holds a valid row; rep(v) = the LOWEST valid row index in it.  spconv keeps one row
 *               per voxel too but leaves open which; fixing the lowest is this op's documented deviation
 *   offset      o = (a * k + c) * k + e, a, c, e in [0, k), delta_o = (a - p, c - p, e - p) over (x, y, z), p = (k-1)/2
 *   out[i]      = bias + sum_o W[:, a, c, e, :] . features[rep(v + delta_o)] for every valid row i in voxel v, summed
 *               over the o whose target voxel is occupied (a cross-correlation, as nn.Conv3d).  Every row of a voxel
 *               gets the same output bit for bit.  Invalid rows get 0 (no bias) and contribute nothing.
 *
 * Backward: exact gradients of the above.  grad_features is the gradient at representative rows and exactly 0 at
 * every other row; grad_weight has weight's layout; grad_bias = sum over valid rows of grad_out.  Any of the three may
 * be NULL (not computed).  fp32 throughout (no TF32), no floating-point atomics: every sum runs in a fixed order
 * (offsets ascending; the rows of a voxel ascending; grad_weight in GF_SUBM_DW_PIECES fixed split-K pieces per offset,
 * summed in piece order), so the output and the three gradients are bit-reproducible from call to call.
 *
 * gf_subm_conv_rulebook builds, from indices alone, the voxel table, the representatives, the [k^3, N] neighbour table,
 * the per-offset pair lists and the rows grouped by voxel; one rulebook serves any number of forward and backward
 * calls on the same indices and desc.  The forward and backward calls also use the workspace for their own scratch,
 * so calls that share a workspace must be ordered (one stream).  Counts stay on the device and the workspace is sized
 * from the desc for the worst case (every row its own voxel), so nothing synchronises and the calls can be captured
 * in a CUDA graph.  With V = batch * X * Y * Z, K = k^3, C = 128 (c_in = c_out), P = GF_SUBM_DW_PIECES, the workspace
 * is, up to 256-byte alignment and a few small arrays,
 *
 *   8 V + 4 N (8 + 2 K + 2 C) + 4 K C^2 (1 + P) bytes
 *
 * (375 MB for N = 144 000 rows on one 200 x 200 x 16 sample with k = 5).  The first uint32 of the workspace is the
 * status word: the rulebook sets GF_FLAG_INDEX_OUT_OF_RANGE when a row is invalid.
 *
 * Supported: c_in = c_out = 128 (GF_ERR_UNSUPPORTED otherwise), odd k <= 5, batch, X, Y, Z, N >= 1; V, N * K and
 * N * C each < 2^31 (GF_ERR_UNSUPPORTED otherwise).  A NULL desc or pointer, an even or larger k, non-positive sizes,
 * indices, features, out, grad_out or grad_features not 16-byte aligned, or a workspace that is NULL, misaligned or
 * smaller than the query fail before any CUDA call. */
#define GF_FLAG_INDEX_OUT_OF_RANGE 16u
#define GF_SUBM_DW_PIECES 8

typedef struct gf_subm_conv_desc {
    int32_t batch;         /* B */
    int32_t num_rows;      /* N */
    int32_t X, Y, Z;       /* spatial shape, over index columns 1, 2, 3 */
    int32_t kernel_size;   /* k: 1, 3 or 5 */
    int32_t c_in, c_out;   /* 128 */
} gf_subm_conv_desc;

size_t gf_subm_conv_workspace_bytes(const gf_subm_conv_desc *desc);

int gf_subm_conv_rulebook(const gf_subm_conv_desc *desc, const int32_t *indices, void *workspace,
                          size_t workspace_bytes, gf_stream_t stream);

int gf_subm_conv_forward(const gf_subm_conv_desc *desc, void *workspace, const float *features, const float *weight,
                         const float *bias, float *out, gf_stream_t stream);

int gf_subm_conv_backward(const gf_subm_conv_desc *desc, void *workspace, const float *features, const float *weight,
                          const float *grad_out, float *grad_features, float *grad_weight, float *grad_bias,
                          gf_stream_t stream);

/* ---- Gaussian refinement: the arithmetic of SparseGaussian3DRefinementModule.forward after its MLP
 * (model/encoder/gaussian_encoder/refine_module.py:72-123, GF_REFINE_V1) and of SparseGaussian3DRefinementModuleV2
 * (refine_module_v2.py:64-108, GF_REFINE_V2), with its gradient.  Inputs: out [B, A, D], the MLP output after mmcv's
 * Scale, D = out_dim = 10 + opa + S (opa = include_opa in {0, 1}, S = semantic_dim), and anchor [B, A, Da].  With the
 * descriptor's constants (the fp32 values the reference's fp32 tensors are combined with):
 *
 *   ssig(v)      = sigmoid(clamp(v, -9.21f, 9.21f))                                                  safe_sigmoid
 *   sinv(t)      = log(t' / (1 - t')),  t' = clamp(t, (float)(1 - 0.9999), 0.9999f)               safe_inverse_sigmoid
 *   normalize(q) = q / max(|q|, 1e-12f)                                                             F.normalize
 *   lo[i] = pc_range[i], extent[i] = (float)(pc_range[i + 3] - pc_range[i])
 *   act          = softmax (max subtracted) | softplus (beta 1, threshold 20: x itself where x > 20) | identity
 *
 * V1 (o = out[b, a], one row):
 *   restrict_xyz:  o[0:3] = (2 ssig(o[0:3]) - 1) * unit      unit[i] = (float)(4 unit_xyz[i] / extent_i), in double
 *   o[0:r] += anchor[0:r]                                    r = refine_prefix (refine_manual must be [0, r))
 *   rot = normalize(o[6:10]);  new_anchor = [o[0:6], rot, o[10:D]]
 * V2:
 *   delta = (2 ssig(out[0:3]) - 1) * unit                    unit = unit_xyz in metres, as the fp32 buffer holds it
 *   orig  = ssig(anchor[0:3]) * extent + lo
 *   axyz  = sinv((orig + delta - lo) / extent)
 *   new_anchor = [axyz, out[3:6], rot, out[10:D]],  rot = normalize(out[6:10]);  o = new_anchor
 * Both:
 *   means     = ssig(o[0:3]) * extent + lo                   (V2: o[0:3] = axyz)
 *   scales    = scale_lo + scale_extent * ssig(o[3:6])
 *   rotations = rot,  opacities = ssig(o[10:10+opa]),  semantics = act(o[10+opa:D])
 *   V2 only:  original_means = orig,  delta_means = delta
 *
 * in fp64 from the fp32 inputs, each output rounded to fp32 once; one thread per anchor.  Shapes: new_anchor [B, A, D],
 * means, scales, original_means, delta_means [B, A, 3], rotations [B, A, 4], opacities [B, A, opa], semantics
 * [B, A, S]; every output the variant has is fully overwritten (original_means and delta_means are ignored by V1).
 *
 * gf_gaussian_refine_backward recomputes the forward from out and anchor and takes the gradient of any subset of the
 * outputs: a NULL gradient counts as zero and is not read.  It fully overwrites grad_out [B, A, D] and grad_anchor
 * [B, A, Da]; grad_anchor is non-zero only in the columns the forward reads (the first r in V1, 0..2 in V2).  The clamps
 * pass the gradient on [lo, hi], bounds included, and block it outside (torch.clamp's backward); normalize follows
 * F.normalize, whose norm below 1e-12f is the constant epsilon; softplus follows PyTorch's threshold.  No atomics: the
 * results are bit-reproducible.  Neither call needs a workspace or synchronises, so both can be captured in a CUDA graph.
 *
 * A NULL desc, negative sizes, an unknown variant or activation, include_opa or restrict_xyz outside {0, 1},
 * out_dim != 10 + include_opa + semantic_dim, a negative refine_prefix or one above min(out_dim, anchor_dim), V2 with
 * refine_prefix or restrict_xyz set or anchor_dim < 3, and NULL pointers for non-empty work are GF_ERR_INVALID_ARG;
 * semantic_dim > GF_REFINE_MAX_SEMANTICS (the semantic logits of an anchor are held in registers) and
 * B * A * max(D, Da) >= 2^31 are GF_ERR_UNSUPPORTED; all before any CUDA call. */
#define GF_REFINE_V1 0
#define GF_REFINE_V2 1
#define GF_REFINE_IDENTITY 0
#define GF_REFINE_SOFTMAX 1
#define GF_REFINE_SOFTPLUS 2
#define GF_REFINE_MAX_SEMANTICS 32

typedef struct gf_refine_desc {
    int32_t variant;                             /* GF_REFINE_V1 | GF_REFINE_V2 */
    int32_t batch, num_anchors, out_dim, anchor_dim;
    int32_t refine_prefix, restrict_xyz;         /* V1 only (0 for V2) */
    int32_t include_opa, semantic_dim, semantics_act;
    float lo[3], extent[3], unit[3];
    float scale_lo, scale_extent;
} gf_refine_desc;

typedef struct gf_refine_outputs {
    float *new_anchor, *means, *scales, *rotations, *opacities, *semantics;
    float *original_means, *delta_means;         /* V2 only */
} gf_refine_outputs;

/* the gradients of the outputs, each NULL (zero) or shaped as its output */
typedef struct gf_refine_grads {
    const float *new_anchor, *means, *scales, *rotations, *opacities, *semantics;
    const float *original_means, *delta_means;
} gf_refine_grads;

int gf_gaussian_refine(const gf_refine_desc *desc, const float *out, const float *anchor,
                       const gf_refine_outputs *outputs, gf_stream_t stream);

int gf_gaussian_refine_backward(const gf_refine_desc *desc, const float *out, const float *anchor,
                                const gf_refine_grads *grads, float *grad_out, float *grad_anchor, gf_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GF_B200_H_ */
