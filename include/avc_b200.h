/* avc_b200.h -- C ABI of libavc_b200.so: H100-native (sm_90a) kernels for the AvatarCLIP
 * appearance-optimisation hot path.
 *
 * The reference (hongfz16/AvatarCLIP, AvatarGen/AppearanceGen) is pure Python/PyTorch and has
 * no FFI layer of its own; the seam it offers is the Python object protocol used by
 * `Runner` (main.py:147-151, 418-420).  Each entry point below replaces the torch-eager
 * implementation of one reference function; the citation names it (paths relative to
 * AvatarGen/AppearanceGen).  INTEGRATION.md shows the ctypes binding a maintainer of the
 * reference would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (a torch tensor), fp32 unless noted;
 *   - every function enqueues work on `stream` and returns immediately (no host sync);
 *   - nothing allocates: scratch is sized by the *_workspace_bytes queries and passed in;
 *   - return value: 0 ok, <0 AVC_E_* (invalid argument), >0 a cudaError_t;
 *   - no results or device state are kept between calls outside the caller's buffers.  Host-side conveniences are
 *     thread-local (a cache of encoded TMA tensor maps, the SM count, "attribute already set" flags): safe to call
 *     from one host thread per device (the supported deployment is one process per GPU, torchrun style).  Tuning
 *     knobs are environment variables (AVC_*, DESIGN.md section 8) read on the host.
 */
#ifndef AVC_B200_H
#define AVC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* avc_stream_t; /* cudaStream_t */

#define AVC_OK 0
#define AVC_E_BADCFG (-1)   /* unsupported network / renderer configuration            */
#define AVC_E_NULL (-2)     /* a required pointer is NULL                               */
#define AVC_E_SIZE (-3)     /* workspace too small / size mismatch                      */
#define AVC_E_ALIGN (-4)    /* pointer not 16-byte aligned                              */
#define AVC_E_NOSTASH (-5)  /* backward called on a workspace with no matching forward  */

#define AVC_ABI_VERSION 3
int avc_abi_version(void);
/* Compiled-for architecture string, e.g. "sm_90a". */
const char* avc_build_arch(void);

/* ------------------------------------------------------------------------------------------
 * NeuS renderer: SDFNetwork + RenderingNetwork + SingleVarianceNetwork + NeuSRenderer.render
 * (models/fields.py:9-107,111-185,270-276; models/embedder.py:6-51; models/renderer.py:39-69,
 * 133-397).  Supported: mode 'no_view_dir', multires_view 0, squeeze_out, weight_norm, n_outside 0 -- i.e.
 * every conf shipped under confs/ (SURVEY.md fact 1).  The kernels always evaluate the extra colour head
 * (extra_color = True, 179 confs); for the one conf without it (base_models/astrongman.conf, --mode train) the host
 * side fills the head's parameter slot with the constant zero map and blends the background into color_fine itself
 * (models/renderer.py:272-281; avatarclip_b200/renderer.py).
 * ------------------------------------------------------------------------------------------ */
typedef struct avc_neus_cfg {
  /* SDFNetwork ctor (models/fields.py:10-21) */
  int32_t sdf_d_in;        /* 3 */
  int32_t sdf_d_out;       /* d_hidden + 1 in every conf: sdf + feature vector */
  int32_t sdf_d_hidden;
  int32_t sdf_n_layers;    /* number of hidden layers; linears = n_layers + 1 */
  uint32_t sdf_skip_mask;  /* bit l set <=> l in skip_in */
  int32_t sdf_multires;
  float sdf_scale;
  /* RenderingNetwork ctor (models/fields.py:112-122); d_in = 6 (points, normals) */
  int32_t col_d_feature;
  int32_t col_d_hidden;
  int32_t col_n_layers;
  /* NeuSRenderer ctor (models/renderer.py:73-93) */
  int32_t n_samples;
  int32_t n_importance;
  int32_t up_sample_steps;
  /* arithmetic engine for the MLP contractions: 0 = fp32 CUDA-core (FFMA) tiles,
   * 1 = wgmma tensor-core tiles with two-term split operands (3 MMAs per product) */
  int32_t engine;
  /* wgmma engine only: MMAs per product in the COLOUR net (forward, dgrad, wgrad).  3 (or 0) = the same two-term split
   * as the SDF trunk; 1 = single-pass bf16 on the hi halves (SURVEY.md Appendix C: the colour net tolerates it in the
   * rendered RGB; the flat parameter gradient moves from ~4e-5 to 3e-4 .. 1e-3 rel-L2, DESIGN.md 3.1). */
  int32_t color_products;
  /* wgmma engine only: MMAs per product in the WEIGHT-GRADIENT tiles (dW += zbar^T in, qt^T ubar, ... : sums over all
   * sample points of a chunk).  3 (or 0) = two-term split operands; 1 = single-pass bf16 on the hi halves. */
  int32_t wgrad_products;
} avc_neus_cfg;

/* Flat parameter vector layout (fp32), identical for the gradient vector:
 *   for each SDF linear l = 0..n_layers:    weight_g[out], weight_v[out*in], bias[out]
 *   for each colour linear l = 0..n_layers: weight_g, weight_v, bias
 *   extra_lin:                              weight_g[3], weight_v[3*d_hidden], bias[3]
 *   variance[1]
 * (the reference's state-dict tensors `linK.weight_g/weight_v/bias`, `extra_lin.*`, `variance`,
 * in named_parameters() order).  avc_neus_param_count returns the total length. */
int avc_neus_param_count(const avc_neus_cfg* cfg, int64_t* n_params);
/* Offset (in floats) of tensor `which` (0 = weight_g, 1 = weight_v, 2 = bias) of linear `layer`
 * of net `net` (0 = sdf, 1 = colour, 2 = extra_lin (layer ignored), 3 = variance). */
int avc_neus_param_offset(const avc_neus_cfg* cfg, int net, int layer, int which, int64_t* offset,
                          int64_t* numel);

/* Bytes of scratch for rendering up to `max_rays_per_chunk` rays per internal chunk. */
int avc_neus_workspace_bytes(const avc_neus_cfg* cfg, int64_t max_rays_per_chunk, size_t* bytes);

typedef struct avc_neus_outputs { /* the dict of models/renderer.py:385-397, all [R, ...] row-major */
  float* color_fine;       /* [R,3]   */
  float* extra_color_fine; /* [R,3]   */
  float* s_val;            /* [R,1]   */
  float* cdf_fine;         /* [R,S]   */
  float* weight_sum;       /* [R,1]   */
  float* weight_max;       /* [R,1]   */
  float* gradients;        /* [R,S,3] */
  float* weights;          /* [R,S]   */
  float* mid_z_vals;       /* [R,S]   */
  float* gradient_error;   /* [1]     */
  float* inside_sphere;    /* [R,S]   */
  float* z_vals;           /* [R,S]  sorted sample depths (saved for the backward) */
} avc_neus_outputs;

/* NeuSRenderer.render forward (models/renderer.py:302-397).
 *   params      flat parameter vector (see above)
 *   rays_o/d    [R,3];  near/far [R]
 *   jitter      [R] values (u-0.5) of renderer.py:317-319, or NULL for perturb = 0
 *   background  NULL, or [3] (bg_kind 1: one colour, main.py:393), or [R] (bg_kind 2: per-ray grey,
 *               main.py:395-405)
 *   z_vals_in   NULL, or [R,S] sorted depths to composite on (skips the placement passes)
 * S = n_samples + n_importance.  The workspace keeps what the backward needs when the call
 * fits one chunk; otherwise the backward recomputes per chunk from out->z_vals. */
int avc_neus_render_fwd(const avc_neus_cfg* cfg, const float* params, const float* rays_o,
                        const float* rays_d, const float* near, const float* far,
                        const float* jitter, const float* background, int bg_kind,
                        const float* z_vals_in, float cos_anneal_ratio, int64_t R,
                        const avc_neus_outputs* out, void* workspace, size_t workspace_bytes,
                        int64_t max_rays_per_chunk, avc_stream_t stream);

typedef struct avc_neus_cotangents { /* d loss / d output; NULL = zero */
  const float* color_fine;       /* [R,3]   */
  const float* extra_color_fine; /* [R,3]   */
  const float* s_val;            /* [R,1]   */
  const float* cdf_fine;         /* [R,S]   */
  const float* weight_sum;       /* [R,1]   */
  const float* weight_max;       /* [R,1]   */
  const float* gradients;        /* [R,S,3] */
  const float* weights;          /* [R,S]   */
  const float* gradient_error;   /* [1]     */
} avc_neus_cotangents;

/* Backward of avc_neus_render_fwd w.r.t. every parameter (the autograd graph the reference builds
 * at models/fields.py:96-107 + main.py:537, second-order terms included).  Overwrites
 * grad_params[n_params].  z_vals / weights etc. are the forward's outputs. */
int avc_neus_render_bwd(const avc_neus_cfg* cfg, const float* params, const float* rays_o,
                        const float* rays_d, const float* background, int bg_kind,
                        float cos_anneal_ratio, int64_t R, const avc_neus_outputs* fwd_out,
                        const avc_neus_cotangents* cot, float* grad_params, void* workspace,
                        size_t workspace_bytes, int64_t max_rays_per_chunk, int32_t flags,
                        avc_stream_t stream);
/* flags for avc_neus_render_bwd: rebuild the forward stash from fwd_out->z_vals even for a
 * single-chunk call (use when the workspace was reused by another call since the forward; the
 * eikonal normaliser is then taken from fwd_out, see DESIGN.md). */
#define AVC_BWD_RECOMPUTE 1

/* SDFNetwork.sdf on arbitrary points (models/fields.py:90-91; used by extract_fields,
 * renderer.py:10-25): sdf_out[P]. */
int avc_neus_sdf_query(const avc_neus_cfg* cfg, const float* params, const float* pts, int64_t P,
                       float* sdf_out, void* workspace, size_t workspace_bytes,
                       avc_stream_t stream);


/* ------------------------------------------------------------------------------------------
 * CLIP ViT-B/32 image tower + cosine loss (openai/CLIP `VisionTransformer`, un-vendored
 * third-party dependency of the reference; call sites main.py:259-261 (load, frozen),
 * :509-526 (resize -> normalise -> encode_image -> cosine against the cached text embedding)).
 * Weights are frozen (main.py:260), so the backward is input-gradient only.
 * GEMM operands are fp16 (clip.load keeps fp16 weights on CUDA), accumulation, the residual
 * stream, LayerNorm and softmax are fp32.
 * ------------------------------------------------------------------------------------------ */
typedef struct avc_clip_cfg {
  int32_t image_size; /* 224 */
  int32_t patch;      /* 32  */
  int32_t width;      /* 768 */
  int32_t layers;     /* 12  */
  int32_t heads;      /* 12  */
  int32_t mlp;        /* 3072 */
  int32_t out_dim;    /* 512 */
} avc_clip_cfg;

typedef struct avc_clip_layer_weights { /* transformer.resblocks.{i}.* ; *_t = transposed copy */
  const float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  const void *w_qkv, *w_qkv_t;   /* fp16 [3W,W], [W,3W]  attn.in_proj_weight  */
  const float* b_qkv;            /* [3W]                 attn.in_proj_bias    */
  const void *w_out, *w_out_t;   /* fp16 [W,W]           attn.out_proj.weight */
  const float* b_out;
  const void *w_fc, *w_fc_t;     /* fp16 [mlp,W], [W,mlp]  mlp.c_fc.weight    */
  const float* b_fc;
  const void *w_proj, *w_proj_t; /* fp16 [W,mlp], [mlp,W]  mlp.c_proj.weight  */
  const float* b_proj;
} avc_clip_layer_weights;

#define AVC_CLIP_MAX_LAYERS 24
typedef struct avc_clip_weights {
  const void *w_patch, *w_patch_t; /* fp16 [W, 3*patch*patch] (conv1.weight flattened), [3*p*p, W] */
  const float *cls, *pos;          /* class_embedding [W], positional_embedding [T,W] */
  const float *ln_pre_g, *ln_pre_b, *ln_post_g, *ln_post_b;
  const float* proj;               /* fp32 [W, out_dim] */
  avc_clip_layer_weights layer[AVC_CLIP_MAX_LAYERS];
} avc_clip_weights;

int avc_clip_workspace_bytes(const avc_clip_cfg* cfg, int32_t B, size_t* bytes);

/* B canvases [B][H][W][3] (fp32, values in [0,1]; the reshape of main.py:510) -> whole-image bilinear
 * resize to image_size^2 (align_corners=False, no antialias) -> Normalize(mean,std) (main.py:261)
 * -> encode_image -> emb_out[B][out_dim]; cos_out[b] = cosine(emb_out[b], text_emb[b]) (main.py:513). */
int avc_clip_loss_fwd(const avc_clip_cfg* cfg, const avc_clip_weights* w, const float* canvases,
                      int32_t H, int32_t W, int32_t B, int32_t input_mode, const float* text_emb,
                      float* emb_out, float* cos_out, void* workspace, size_t workspace_bytes,
                      avc_stream_t stream);
/* input_mode 0: canvases as above.  input_mode 1: `canvases` is an already resized + normalised NCHW
 * image batch [B][3][image_size][image_size] (the argument of perceptor.encode_image, main.py:512);
 * H = W = image_size.
 * Backward: d loss / d input given g_cos[b] = d loss / d cos_out[b] and/or g_emb[b][out_dim] =
 * d loss / d emb_out (either may be NULL); uses what the forward left in the workspace.  Overwrites
 * d_canvases (same shape as the forward input). */
int avc_clip_loss_bwd(const avc_clip_cfg* cfg, const avc_clip_weights* w, int32_t H, int32_t W, int32_t B,
                      int32_t input_mode, const float* text_emb, const float* g_cos, const float* g_emb,
                      float* d_canvases, void* workspace, size_t workspace_bytes, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * CLIP ViT-B/32 text tower (openai/CLIP `CLIP.encode_text`, the prompt embeddings of main.py:276,282,288; the
 * weights are the non-`visual.*` half of ViT-B-32.pt).  Forward only: the weights are frozen and the reference
 * detaches the embedding.  token_embedding + positional_embedding, `layers` pre-LN residual blocks with causal
 * self-attention (scale 1/sqrt(64), fp32 softmax) and QuickGELU MLP, ln_final on the row of each sequence's first
 * maximal token id (<|endoftext|>), @ text_projection.  Same precision scheme as the image tower: fp16 GEMM operands,
 * fp32 accumulation, residual stream, LayerNorm and softmax.  Supported: width / heads == 64, width <= 1024,
 * context <= 128, mlp % 64 == 0, 1 <= layers <= AVC_CLIP_MAX_LAYERS; anything else is AVC_E_BADCFG.
 * ------------------------------------------------------------------------------------------ */
typedef struct avc_clip_text_cfg {
  int32_t context;    /* 77    */
  int32_t vocab;      /* 49408 */
  int32_t width;      /* 512   */
  int32_t layers;     /* 12    */
  int32_t heads;      /* 8     */
  int32_t mlp;        /* 2048  */
  int32_t out_dim;    /* 512   */
} avc_clip_text_cfg;

typedef struct avc_clip_text_weights {
  const float* token_emb;          /* [vocab, W]  token_embedding.weight (fp16 values stored as fp32) */
  const float* pos;                /* [context, W] positional_embedding (fp16 values stored as fp32) */
  const float *ln_final_g, *ln_final_b;
  const float* proj;               /* fp32 [W, out_dim] text_projection */
  /* transformer.resblocks.{i}.*: the forward reads w_qkv / w_out / w_fc / w_proj, the biases and the LayerNorms;
   * the transposed copies (*_t) are unused and may be NULL */
  avc_clip_layer_weights layer[AVC_CLIP_MAX_LAYERS];
} avc_clip_text_weights;

int avc_clip_text_workspace_bytes(const avc_clip_text_cfg* cfg, int32_t B, size_t* bytes);
/* tokens: DEVICE int32 [B][context] (clip.tokenize); ids must lie in [0, vocab) -- an id outside is clamped, never read
 * out of bounds.  emb_out[B][out_dim] = encode_text(tokens). */
int avc_clip_encode_text(const avc_clip_text_cfg* cfg, const avc_clip_text_weights* w, const int32_t* tokens, int32_t B,
                         float* emb_out, void* workspace, size_t workspace_bytes, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Shading + canvas scatter + non-CLIP losses of Runner.train_clip (main.py:417-497, 528-534) with
 * use_silhouettes = True (every shipped train_clip conf).  The two switches the shipped confs vary
 * (the 18 confs/ablation files ending in _0 / _1 / _2) are the last two fields: zero-initialised = add_no_texture = texture_cast_light =
 * True, the configuration of confs/examples*.
 * Rays are the True pixels of the dilated mask; pix[r] is the flat canvas index (y*W + x) of ray r.
 * ------------------------------------------------------------------------------------------ */
typedef struct avc_loss_inputs {
  /* render outputs (NeuSRenderer.render dict) */
  const float* color_fine;       /* [R,3] */
  const float* extra_color_fine; /* [R,3] */
  const float* gradients;        /* [R,S,3] */
  const float* weights;          /* [R,S] */
  const float* weight_sum;       /* [R] */
  const float* gradient_error;   /* [1] */
  /* per step */
  const int32_t* pix;            /* [R] canvas index of each ray */
  const uint8_t* in_mask;        /* [H*W] 1 where a ray exists (the dilated mask, dataset.py:255-256) */
  const float* true_rgb;         /* [H*W,3] template render resized to the canvas (main.py:376) */
  const float* mask;             /* [H*W] 0/1 (main.py:377-380, 407-410) */
  const float* background;       /* NULL, or [H*W] grey levels for bg_choice 1/2 (main.py:394-405) */
  int32_t bg_choice;             /* 0 white, 1/2 per-pixel grey, 3 black (main.py:387-415) */
  float light_dir[3];            /* sphere_coord(theta+U, phi+U) of main.py:433 (un-normalised) */
  float ambience;                /* main.py:440 */
  const float* view_scalars;     /* NULL, or DEVICE [4] = {light_dir[3], ambience}: overrides the two host fields above
                                    (lets a captured CUDA graph of the step be replayed with new per-view draws) */
  float igr_weight, mask_weight, clip_weight;  /* conf train.* */
  int32_t R, S, H, W;
  /* ABI 3 */
  int32_t plain_texture;         /* 1: train.texture_cast_light = False -- canvas 0 is the extra colour itself
                                    (full_extra_color_fine, main.py:475-477,516), no shading factor, no clamp */
  int32_t no_shading_term;       /* 1: train.add_no_texture = False -- the loss has no CLIP term on canvas 1
                                    (main.py:521,533): the backward ignores d_canvases[1] */
} avc_loss_inputs;

/* scalars written by the forward: [0] color_loss, [1] eikonal, [2] mask_loss (BCE), [3] psnr,
 * [4] base_loss = color + igr*eik + mask_w*bce, [5..7] internal sums (l1, bce, sq), [8] mask_sum */
#define AVC_LOSS_SCALARS 16
/* Forward: fills canvases[2][H][W][3] (0: texture_shading -- or the extra colour when plain_texture --,
 * 1: rand_shading_rgb; main.py:466-477) and scalars[AVC_LOSS_SCALARS].  Canvas 1 is always written (finite values)
 * so that a caller may keep one B = 2 CLIP batch for every configuration. */
int avc_loss_stage_fwd(const avc_loss_inputs* in, float* canvases, float* scalars, avc_stream_t stream);
/* Backward: d_canvases[2][H][W][3] = d loss / d canvases (from the CLIP backward) plus the direct
 * loss terms -> cotangents of the render outputs (struct avc_neus_cotangents, written in full:
 * color_fine, extra_color_fine, gradients, weights, weight_sum, gradient_error must be non-NULL
 * writable buffers; s_val, cdf_fine, weight_max are ignored). */
int avc_loss_stage_bwd(const avc_loss_inputs* in, const float* d_canvases, const float* scalars,
                       const avc_neus_cotangents* cot_out, avc_stream_t stream);

/* SDFNetwork.forward / .sdf_hidden_appearance / .gradient (models/fields.py:72-107) on P arbitrary points (boundary
 * convenience, exact-fp32 tiles regardless of cfg->engine): sdf_feat_out [P][d_out] = (sdf, feature vector) or NULL;
 * grad_out [P][3] = d sdf / d x (raw, un-normalised) or NULL.  Workspace: as avc_neus_sdf_query. */
int avc_neus_sdf_eval(const avc_neus_cfg* cfg, const float* params, const float* pts, int64_t P, float* sdf_feat_out,
                      float* grad_out, void* workspace, size_t workspace_bytes, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused Adam over the flat parameter vector (torch.optim.Adam defaults, main.py:145,536-538):
 * p -= lr * mhat / (sqrt(vhat) + eps); `step` is the 1-based step count; grad_scale multiplies g
 * first (1/world_size after the gradient all-reduce).
 * ------------------------------------------------------------------------------------------ */
int avc_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                  float lr, float beta1, float beta2, float eps, int64_t step, float grad_scale,
                  avc_stream_t stream);
/* Same update with the step counter and the learning rate in DEVICE memory, so that the call can be captured
 * once in a CUDA graph and replayed: state[0] = step count so far (incremented by the call), state[1] = lr
 * (written by the host before each replay), state[2..3] = scratch. */
int avc_adam_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                      float* state, float beta1, float beta2, float eps, float grad_scale, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Camera rays: SMPL_Dataset.gen_rays_pose / gen_rays_silhouettes + near_far_from_sphere
 * (models/dataset.py:252-293, 331-342).  pose_c2w is a HOST pointer to the 4x4 row-major camera-to-world matrix
 * (lookat, models/utils.py:9-27).  Pixel grid: linspace(0, full-1, W) x linspace(0, full-1, H).  pix[R] lists the
 * selected canvas pixels (y*W + x; the True entries of the dilated mask) or is NULL for all W*H pixels.
 * ------------------------------------------------------------------------------------------ */
int avc_gen_rays(const float* pose_c2w, float fx, float fy, float cx, float cy, int32_t full_w, int32_t full_h,
                 int32_t W, int32_t H, const int32_t* pix, int32_t R, float* rays_o, float* rays_d, float* near,
                 float* far, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * SMPL linear-blend skinning: my_lbs(v_shaped, pose, v_template, shapedirs, posedirs, J_regressor, parents,
 * lbs_weights, pose2rot) of models/utils.py:176-224 (batch 1; v_template / shapedirs are unused by the reference
 * function and therefore absent here).  pose: [n_joints*3] axis-angle when pose2rot != 0, else [n_joints][3][3]
 * rotation matrices.  posedirs: [(n_joints-1)*9][V*3].  lbs_weights: [V][n_joints].  n_joints <= 32.
 * Outputs: verts_out [V][3], joints_out [n_joints][3] (J_transformed).
 * ------------------------------------------------------------------------------------------ */
int avc_lbs_workspace_bytes(int32_t n_joints, size_t* bytes);
int avc_lbs_fwd(const float* v_shaped, const float* pose, int32_t pose2rot, const float* J_regressor,
                const int32_t* parents, const float* posedirs, const float* lbs_weights, int32_t V,
                int32_t n_joints, float* verts_out, float* joints_out, void* workspace,
                size_t workspace_bytes, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Mesh animation: AvatarGen/AppearanceGen/drive.py (generate_animation :308-361), the step after validate_mesh that
 * rigs the exported mesh with SMPL skin weights and skins it through a motion.  Indices are int32, points fp32.
 *
 * avc_nearest_vertex replaces find_nearest_ind (drive.py:235-240): nearest[i] = argmin_j ((ref[j] - query[i])**2).sum()
 * in fp64 -- each operand promoted exactly, the sum taken as (dx*dx + dy*dy) + dz*dz without fused multiply-adds, as
 * numpy does -- ties to the smallest j.  query [N][3], ref [M][3], nearest [N].
 * ------------------------------------------------------------------------------------------ */
int avc_nearest_vertex(const float* query, int32_t N, const float* ref, int32_t M, int32_t* nearest,
                       avc_stream_t stream);

/* Replaces the island search of cleanup_mesh (drive.py:172-203; the removal :204-209 is the caller's gather).
 * Components of the graph whose edges are the triangle edges; a vertex in no triangle is a component of its own.
 * faces [F][3] (F may be 0; a triangle with an index outside [0, V) is ignored).  labels [V]: the smallest vertex
 * index of each vertex's component.  kept [2] (DEVICE): {label, size} of the largest component; among equal sizes the
 * one with the smallest label, i.e. the first the reference's scan in vertex order finds.  Nothing is read back to the
 * host.  Workspace: avc_mesh_components_workspace_bytes(V). */
int avc_mesh_components_workspace_bytes(int32_t V, size_t* bytes);
int avc_mesh_components(const int32_t* faces, int32_t F, int32_t V, int32_t* labels, int32_t* kept, void* workspace,
                        size_t workspace_bytes, avc_stream_t stream);

/* The joint transforms of inv_lbs / lbs (drive.py:243-245, 256-258) with beta = 0, for n_frames poses at once:
 * joints_out [n_joints][3] = J_regressor . v_template (vertices2joints, :51-68); A_out [n_frames][n_joints][3][4] =
 * the top three rows of batch_rigid_transform's rel_transforms (:93-148; the bottom row is [0 0 0 1]).  pose:
 * [n_frames][n_joints][3] axis-angle when pose2rot != 0 (batch_rodrigues, :13-49), else [n_frames][n_joints][3][3]
 * rotation matrices.  v_template [V][3], J_regressor [n_joints][V], parents [n_joints] (parents[0] = -1, a parent
 * before its child).  1 <= n_joints <= 32. */
int avc_lbs_rel_transforms(const float* v_template, const float* J_regressor, const int32_t* parents, int32_t V,
                           int32_t n_joints, const float* pose, int32_t pose2rot, int32_t n_frames, float* joints_out,
                           float* A_out, avc_stream_t stream);

/* inv_lbs (drive.py:242-253): per vertex T = sum_j W[v][j] A_j as a 4x4 whose bottom row is [0 0 0 s], s = sum_j
 * W[v][j]; tpose_out[v] = rows 0-2 of T^-1 . [verts[v]; 1] = M^-1 (p - t / s) for T's top block [M | t], in fp64.
 * W[v] = lbs_weights[nearest[v]] (the gather of drive.py:338-339), or lbs_weights[v] when nearest is NULL (then
 * M >= N).  verts [N][3], lbs_weights [M][n_joints], A [n_joints][3][4] (one frame of avc_lbs_rel_transforms). */
int avc_inv_lbs(const float* verts, const int32_t* nearest, int32_t N, const float* lbs_weights, int32_t M,
                int32_t n_joints, const float* A, float* tpose_out, avc_stream_t stream);

/* lbs (drive.py:255-265, no pose blend shapes) over frames [frame_begin, frame_begin + frame_count) of A
 * [n_frames][n_joints][3][4]: out[f - frame_begin][v] = (sum_j W[v][j] A[f]_j) . [tpose[v]; 1], i.e. the float32
 * payload of write_pc2 (:295-305) for those frames.  W as in avc_inv_lbs. */
int avc_lbs_frames(const float* tpose, const int32_t* nearest, int32_t N, const float* lbs_weights, int32_t M,
                   int32_t n_joints, const float* A, int32_t n_frames, int32_t frame_begin, int32_t frame_count,
                   float* out, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Avatar export: Avatar2FBX/export_fbx.py (:44-118), which rigs the exported mesh to SMPL's skeleton.
 *
 * avc_nearest_vertex_f32 is Avatar2FBX's find_nearest_ind (utils/ply_utils.py:84-89), where both operands are float32:
 * nearest[i] = argmin_j of the float32 (dx*dx + dy*dy) + dz*dz, d = ref[j] - query[i], every operation rounded on its
 * own (no fused multiply-adds), ties to the smallest j.  Near-equidistant reference points may give another index than
 * avc_nearest_vertex's fp64 distance.  Shapes and errors as avc_nearest_vertex.
 * ------------------------------------------------------------------------------------------ */
int avc_nearest_vertex_f32(const float* query, int32_t N, const float* ref, int32_t M, int32_t* nearest,
                           avc_stream_t stream);

/* open3d's TriangleMesh::simplify_vertex_clustering(voxel, SimplificationContraction.Average) with Avatar2FBX's voxel
 * (utils/ply_utils.py:16-19): voxel = max over axes of (max - min) / resolution (resolution 256 there).
 *   - Voxel of a vertex: idx = floor((v - (min - voxel / 2)) / voxel) per axis, in fp64 with each operation rounded on
 *     its own, so a vertex exactly on a voxel boundary lands where numpy / Eigen put it.  If every vertex is the same
 *     point (voxel 0) they share one voxel.
 *   - Output vertex k is the k-th distinct voxel in order of its first vertex, scanning the input in index order.
 *     Vertices in no triangle are clustered too.
 *   - Its position is the fp64 mean of the voxel's positions, rounded to float32; its colour (when colors is not NULL)
 *     the fp64 mean of c / 255, rounded to float32.  The sums are taken by atomics in no fixed order.  They are exact,
 *     so the means do not depend on that order, whenever the sum of a voxel's coordinates fits in 53 bits: its values
 *     lie on one power-of-two grid no finer than about 2^-29 of their magnitude (true of the avatar meshes measured; a
 *     coordinate of 1e-16 beside one of 1e-2 is not, and such a voxel may change in its last bit between runs).
 *     Colours are summed as integers and may differ from a sequential fp64 mean of c / 255 by one float32 ulp.
 *   - Triangles are remapped in input order.  A triangle with two corners in one voxel is dropped, and so is one that
 *     is a rotation (a,b,c), (b,c,a) or (c,a,b) of an earlier kept triangle; a reversed triangle (a,c,b) is kept.  A
 *     kept triangle keeps the rotation it first appeared in.  A triangle with an index outside [0, V) is dropped.
 * verts [V][3], colors [V][3] uint8 or NULL, tris [F][3] (F may be 0).  Outputs sized by the inputs: verts_out [V][3],
 * colors_out [V][3] (required when colors is given), tris_out [F][3].  counts [2] (DEVICE): {output vertices, output
 * triangles}; the rows beyond them are left unwritten.  Nothing is read back to the host.  1 <= resolution <=
 * 2^21 - 2 (the voxel key packs 21 bits per axis), else AVC_E_BADCFG.  1 <= V <= 2^30, 0 <= F <= 2^30.
 * Workspace: avc_mesh_cluster_workspace_bytes(V, F). */
int avc_mesh_cluster_workspace_bytes(int32_t V, int32_t F, size_t* bytes);
int avc_mesh_cluster(const float* verts, const uint8_t* colors, int32_t V, const int32_t* tris, int32_t F,
                     int32_t resolution, float* verts_out, float* colors_out, int32_t* tris_out, int32_t* counts,
                     void* workspace, size_t workspace_bytes, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Self-test of the wgmma GEMM tiles (engine 1): C[M][N] = A[M][K] . B[N][K]^T, fp32 in/out, operands
 * split into bf16 (hi, lo) pairs; nprod = 1 (hi*hi only) or 3 (hi*hi + hi*lo + lo*hi).
 * workspace >= 4 * (M + N) * round_up(K, 8) + 1024 bytes.
 * ------------------------------------------------------------------------------------------ */
int avc_tc_gemm_nt_test(const float* A, const float* B, int64_t M, int32_t N, int32_t K, int32_t nprod,
                        float* C, void* workspace, size_t workspace_bytes, avc_stream_t stream);
/* Same for the reduction-over-rows tiles (weight gradients): C[N1][N2] += A[P][N1]^T . B[P][N2]; when colsum is not
 * NULL also colsum[N1] += column sums of A (the fused bias gradient).
 * workspace >= 4 * P * (round_up(N1,8) + round_up(N2,8)) + 2048 bytes. */
int avc_tc_gemm_tn_test(const float* A, const float* B, int64_t P, int32_t N1, int32_t N2, int32_t nprod,
                        float* C, float* colsum, void* workspace, size_t workspace_bytes, avc_stream_t stream);
/* 1: the last wgmma NT launch of the calling host thread stored its outputs with TMA bulk stores through the epilogue
 * ring, 0: from registers, -1: no launch yet (the tests check which path a shape takes). */
int avc_tc_nt_last_ring(void);
/* The backward epilogue functors of the NeuS path through the NT tiles on caller data: kind 0 second-order sweep,
 * 1 / 2 value backward without / with the sdf term, 3 gradient chain, 4 ReLU-mask dgrad, 5 encoding-gradient
 * accumulation; and with the bf16 split of their output: 6 value chain, 7 feature bias, 8 colour lin0, 9 ReLU,
 * 10 plain store, 11 ReLU-mask dgrad, 108..111 as 8..11 with one bf16 product; and with the output sets the renderer
 * gives them: 12 second-order sweep with the split of ubar, 13 / 14 value backward with only the split of the new
 * zbar_prev, without / with the sdf term, 15 gradient chain with only the split of qt_prev (argument roles in avc_neus.cu).
 * workspace >= 4 * (M + N) * round_up(K, 8) + 4 * M * ldx bytes. */
int avc_tc_epi_test(int32_t kind, const float* A, const float* B, int64_t M, int32_t N, int32_t K, int32_t Nv,
                    const float* X, float* Y, int32_t ldx, const float* v1, const float* v2, float s, float s2, float* OUT,
                    float* OUT2, int32_t ld2, void* workspace, size_t workspace_bytes, avc_stream_t stream);
/* One kernel of the NeuS path outside the GEMM tiles (avc_neus_kernels.cuh) on caller buffers, launched by the
 * host helpers the render uses.  dims is a HOST int64 array, fscal a HOST float array, in / out HOST arrays of DEVICE
 * pointers (all fp32).  An input marked "or NULL" may be NULL exactly where the render passes NULL.  ctx is the [4+]
 * scalar block {inv_s, eik_num, eik_den, invs_bar}; the kinds add into its sums as the render does.
 *   0 k_ctx_init       dims {off_var, zero_sums};  in {params};  out {ctx}
 *   1 k_composite_fwd + k_reduce_ray_part (eik_num, eik_den)   dims {S <= 256, Rc, bg_kind};  fscal {cos_anneal,
 *     sample_dist};  in {rays_d[Rc][3], z[Rc][S], sdf[P], cin[P][8], rgb6[P][8], background ([3] | [Rc] | NULL)};
 *     out {color[Rc][3], extra[Rc][3], s_val[Rc], cdf[P], wsum[Rc], wmax[Rc], weights[P], ray_part[Rc][4], ctx}
 *   2 k_composite_bwd + k_reduce_ray_part (invs_bar)   dims, fscal as 1;  in {as 1, then the cotangents g_color[Rc][3],
 *     g_extra[Rc][3], g_wsum[Rc], g_wmax[Rc], g_w[P], g_cdf[P], g_n[P][3], g_gerr[1] (each or NULL), weights[P] (or NULL
 *     when g_wmax is)};  out {y6bar[P][8], sdfbar[P], nbar[P][4], ray_part[Rc][4], ctx}
 *   3 k_relax_count + k_reduce_ray_part (eik_den)   dims {S, Rc};  fscal {sample_dist};  in {rays_o, rays_d, z[Rc][S]};
 *     out {ray_part[Rc][4], ctx}
 *   4 k_finalize_fwd   in {ctx};  out {gradient_error[1]}
 *   5 k_variance_grad  dims {off_var, R};  in {params, ctx, g_sval[R] or NULL};  out {grad_var[1]}
 *   6 k_coarse_z       dims {n, pitch, Rc};  in {near[Rc], far[Rc], jitter[Rc] or NULL};  out {z[Rc][pitch]}
 *   7 k_upsample       dims {n (2..256), pitch, Rc, per (1..64)};  fscal {inv_s};  in {rays_o, rays_d, z[Rc][pitch],
 *     sdf[Rc][pitch]};  out {newz[Rc][per]}
 *   8 k_merge          dims {n (<= 256), pitch, Rc, per (<= 64), pitch_o >= n + per};  in {z[Rc][pitch], sdf[Rc][pitch],
 *     newz[Rc][per], news[Rc][per] or NULL};  out {zo[Rc][pitch_o], so[Rc][pitch_o] (unused when news is NULL)}
 * A "pair" output is the two-term bf16 split of a [rows][ld] activation as ONE bf16 buffer [rows][2 ld]: hi in columns
 * [0, ld), lo in [ld, 2 ld) of each row; NULL where the render passes no split.  Kinds 9..11, 15..17, 20..24 and 26 run
 * on a whole configuration: in[0] is a HOST avc_neus_cfg, the widths and pitches below are those of its plan (K_l, Kp_l,
 * Np_l of SDF linear l; E, EP the encoded width and its pitch; Hc, F), pack is what kind 10 writes.  dims[0] = P.
 *   9 pack layout       out {HOST int64 [16 + 11 (L + Lc + 3)]}: {L, Lc, E, EP, F, Fp, Hc, pack_floats, n_params,
 *     off_var, pk_wsdf, pk_bsdf, pk_c0x, pk_c0xT, pk_W6, pk_b6}, then per SDF linear 0..L, colour linear 0..Lc and
 *     extra_lin: {K, N, Kp, Np, skip, off_g, off_v, off_b, pk_W, pk_WT, pk_b}
 *  10 prepare_weights   in {cfg, params};  out {pack[pack_floats], engine 1: pk pair [2 pack_floats] (hi, then lo)}
 *  11 k_wn_backward     in {cfg, params, wbar[n_params]};  out {grads[n_params]} (the g / v / bias slots of every linear)
 *  12 k_encode_points, 13 k_encode_samples, 14 k_encode_fine: dims {multires, ld0, n_skip (<= 4), skip_ld[4],
 *     skip_col[4], then 12: P; 13: nz, pitch, Rc; 14: S, Rc};  fscal {scale, 14: sample_dist};  in {12: pts[P][3];
 *     13: rays_o, rays_d, z[Rc][pitch]; 14: rays_o, rays_d, z_vals[Rc][S]};  out {in0[P][ld0] or NULL, skip[4] fp32
 *     [P][skip_ld] or NULL, in0 pair or NULL, skip pairs[4] or NULL, 14: cin[P][8], mid_z[P] or NULL, inside[P] or NULL}
 *  15 k_thin_nt<1, OutSdf> (value chain's sdf head)  dims {P, nz, pitch};  in {cfg, in_L[P][Kp_L], pack};  out {sdf}
 *  16 k_thin_nt<6, OutHeads>   in {cfg, ch[P][Hc], pack};  out {rgb6[P][8]}
 *  17 k_thin_nt<6, OutNbarAdd> in {cfg, cbar[P][Hc], pack};  out {nbar[P][4] (added into)}
 *  18 k_thin_tn<NI>     dims {NI (1 | 6), lds, ldh, NC, P, si, sc, split};  fscal {s_scale};  in {S[P][lds], Hm[P][ldh]};
 *     out {out, bout or NULL, out2 or NULL, bout2 or NULL} (added into)
 *  19 k_colsum          dims {ld, NC, P};  fscal {scale};  in {X[P][ld]};  out {out[NC] (added into)}
 *  20 k_heads_dgrad     in {cfg, y6bar[P][8], pack, ch[P][Hc]};  out {cbar[P][Hc] or NULL, pair or NULL}
 *  21 k_chain_start     in {cfg, pack, sp'(z)[P][Np_{L-1}]};  out {qt[P][Np_{L-1}] or NULL, ge[P][EP], pair or NULL}
 *  22 k_normal          in {cfg, ge[P][EP]};  out {cin[P][8] (x read from 0:3, n written to 3:6), grad[P][3] or NULL}
 *  23 k_dge             in {cfg, cin[P][8], nbar[P][4]};  out {ubar0[P][Kp_0] or NULL, gebar[P][EP], pair or NULL}
 *  24 k_fill_gebar      dims {P, l (a skip layer)};  in {cfg, gebar[P][EP]};  out {ubar_l[P][Kp_l], pair or NULL}
 *  25 k_points_to_cin   dims {P};  in {pts[P][3]};  out {cin[P][8]}
 *  26 k_assemble_sdf_feat  in {cfg, sdf[P], feat[P][Fp]};  out {[P][F + 1]} */
int avc_neus_kernel_test(int32_t kind, const int64_t* dims, const float* fscal, const void* const* in, void* const* out,
                         avc_stream_t stream);
/* One kernel of the CLIP towers (avc_clip.cu) on caller buffers, launched by the host code the towers use (the GEMMs
 * through the same M <= 128 wgmma / M > 128 mma.sync dispatch and split-K recomputation).  dims is a HOST int array,
 * in / out are HOST arrays of DEVICE pointers; "h" marks fp16, "i" int32, everything else is fp32.  Outputs are
 * written in place (x, dst, dy, dx are read as well when the kernel accumulates).  Nothing else is touched.
 *   0..6 GEMM  acc[M][N] = A[M][K] . Wt[N][K]^T, dims {M, N, K, ksplit (, np)}; in {A h, Wt h, aux}:
 *        0 out[0][M][N]  = acc + bias(aux[N])                          (EpiBiasStore)
 *        1 out[0][M][N] += acc + bias(aux[N]) once over the splits      (EpiResidual)
 *        2 out[0][M][N]  = pre = acc + bias(aux[N]), out[1] h = QuickGELU(pre)     (EpiFc)
 *        3 out[1] h[M][N] = acc * QuickGELU'(pre), pre = aux[M][N]                 (EpiDfc)
 *        4 out[0][M][N] += acc / aux[M]                                 (EpiAccumUnscale)
 *        5 out[0][M][N]  = acc / aux[M]                                 (EpiStoreUnscale)
 *        6 out[0][b*(np+1) + 1 + p][N] += acc[b*np + p]                 (EpiPatch; aux unused)
 *   7  k_layernorm      dims {M, Wd};  in {x, g, b};  out {y32, y16 h, save_x}, any may be NULL
 *   8  k_layernorm_bwd  dims {M, Wd, accumulate, zero_dy};  in {x, g};  out {dy, dx, dx16 h or NULL, dx_scale[M]}
 *   9  k_to_half_rowscaled  dims {M, N, ld_src};  in {src, row_map i[M] or NULL};  out {dst h[M][N], scale[M]}
 *   10 k_attention      dims {B, T, Wd, heads};  in {qkv[B*T][3Wd]};  out {o16 h[B*T][Wd]}
 *   11 k_attention_bwd  dims {B, T, Wd, heads};  in {qkv, dO[B*T][Wd]};  out {dqkv[B*T][3Wd]}
 *   12 k_causal_attention  dims {B, T, Wd, heads};  in {qkv};  out {o16 h}
 *   13 k_preprocess     dims {H, W, B, IS, P, mode};  in {canvas};  out {a0 h[B*(IS/P)^2][3P^2]}
 *   14 k_preprocess_bwd dims as 13;  in {dpatch};  out {dcanvas} (zeroed first)
 *   15 k_head_proj      dims {B, T, Wd, OD};  in {x[B*T][Wd], g, b, proj[Wd][OD]};  out {emb[B][OD], ynorm[B][Wd]}
 *   16 k_cosine         dims {B, OD};  in {emb, text};  out {cos[B]}
 *   17 k_head_bwd_dy    dims {B, Wd, OD};  in {proj, text, emb, g_cos[B] or NULL, g_emb[B][OD] or NULL};  out {dy[B][Wd]}
 *   18 k_head_bwd_ln    dims {B, T, Wd};  in {x[B*T][Wd], g, dy[B][Wd]};  out {dx[B*T][Wd]}
 *   19 k_text_eot_rows  dims {B, T, Wd};  in {tok i[B][T], x[B*T][Wd]};  out {eot[B][Wd]} */
int avc_clip_kernel_test(int32_t kind, const int32_t* dims, const void* const* in, void* const* out,
                         avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Per-step view preparation of Runner.train_clip (SURVEY.md 8f rank 1), all on the device.
 *
 * avc_raster_template replaces render_one_batch (models/utils.py:108-125 -> neural_renderer Renderer(camera_mode=
 * 'look'), image_size 256, 2x anti-aliasing, white textures, ambient 0.5 + directional 0.5 along +y, fill_back):
 * verts [V][3] (SMPL frame; the (x, z, -y) re-orientation of utils.py:115-119 happens inside), faces [F][3] int32,
 * eye / at [3] HOST pointers; rgb_out [n][n][3] already flipped like utils.py:124; mask_out [n][n] = (rgb != 0)
 * (main.py:361-364).  avc_dilate_count = ndimage.binary_dilation(mask, 3x3 full structure, iterations) and the
 * pixel count that sizes the canvas (models/dataset.py:255-258).  avc_mask_compact = nearest resize of the dilated
 * mask to W x W (F.interpolate default) + the row-major list of its True pixels (dataset.py:269-273); pix holds at
 * most `cap` entries, count_out the true count.  avc_view_targets = main.py:375-380,407-410 (nearest resize of the
 * template render, mask = channel 0 != 0, or all ones when threshold_mask == 0 i.e. mask_weight == 0).
 * avc_background_field = main.py:392-402: kind 1 clamp(N(0.5, 0.2), 0, 1) per pixel, kind 2 the 0.2 / 0.8
 * chessboard of chess_len-pixel squares blurred by GaussianBlur(kernel (5, 9), sigma); optional gather to the rays
 * (main.py:412-413).  avc_uniform_fill: counter-based U[lo, hi) draws (per-ray jitter, renderer.py:317-319).
 * ------------------------------------------------------------------------------------------ */
int avc_raster_workspace_bytes(int32_t V, int32_t image_size, int32_t supersample, size_t* bytes);
int avc_raster_template(const float* verts, const int32_t* faces, int32_t V, int32_t F, const float* eye,
                        const float* at, int32_t image_size, int32_t supersample, float* rgb_out, uint8_t* mask_out,
                        void* workspace, size_t workspace_bytes, avc_stream_t stream);
int avc_dilate_count(const uint8_t* mask, int32_t n, int32_t iterations, uint8_t* dilated, int32_t* count_out,
                     avc_stream_t stream);
int avc_mask_compact(const uint8_t* dilated, int32_t n, int32_t W, int32_t cap, uint8_t* in_mask, int32_t* pix,
                     int32_t* count_out, avc_stream_t stream);
int avc_view_targets(const float* rgb, int32_t n, int32_t W, int32_t threshold_mask, float* true_rgb, float* mask,
                     avc_stream_t stream);
int avc_background_field(int32_t kind, int32_t H, int32_t W, uint32_t seed, int32_t chess_len, float sigma,
                         float* canvas_bg, const int32_t* pix, int32_t R, float* ray_bg, avc_stream_t stream);
int avc_uniform_fill(uint32_t seed, int32_t n, float lo, float hi, float* out, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Iso-surface extraction for NeuSRenderer.extract_geometry (models/renderer.py:27-36,399-404; the reference calls
 * PyMCubes' marching_cubes, third-party, absent).  Marching tetrahedra over the [nx][ny][nz] field u (= -sdf):
 * avc_march_count writes the number of triangles of every grid cube ((nx-1)(ny-1)(nz-1) ints, x-major like the
 * field); the caller turns them into exclusive offsets; avc_march_emit writes 3 vertices per triangle in INDEX
 * coordinates (the caller rescales like renderer.py:33-35) and, per vertex, a 64-bit key of the grid edge it lies
 * on (for welding).  Triangles are oriented with normals towards decreasing u.
 * ------------------------------------------------------------------------------------------ */
/* Profiling aid of the fused value-chain kernel: with AVC_CHAIN_DEBUG=1 in the environment block 0 records cycle
 * counters ([0] MMA warp waiting for its A operand, [1] for weight slabs, [2] MMA warp total, [3] tile-layers,
 * [4] epilogue waiting for the accumulator, [5] epilogue work); this call synchronises the device and copies them. */
int avc_chain_debug_read(long long* out8);
/* Stall probe of the wgmma NT tiles: only in a diagnostic build (-DAVC_NT_PROBE=1, tools/nt_probe.py); a regular
 * build returns AVC_E_BADCFG.  host_out[16][10]: per epilogue functor the summed cycles {producer waiting for a free
 * stage, producer loop, consumers waiting for operands, consumers waiting for their turn, consumers' MMAs, consumers'
 * epilogues, consumers' loops, CTAs, consumers waiting for staged epilogue operands, consumers waiting for their TMA
 * stores to release a ring slot} (consumer slots: both consumer warpgroups); reset != 0 clears the counters. */
int avc_nt_probe_read(unsigned long long* host_out, int reset);

int avc_march_count(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, int32_t* counts,
                    avc_stream_t stream);
int avc_march_emit(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, const int32_t* offsets,
                   float* verts, int64_t* keys, avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * ShapeGen: the coarse body shape from a text prompt (AvatarGen/ShapeGen/main.py:93-123, utils.py:9-35).
 *
 * avc_vae_decode is LinearVAE.decode (main.py:67-68): out[b][D] = W2[D][H] . (W1[H][L] . z[b][L] + b1[H]) + b2[D] +
 * v_template[D] for 1 <= B <= 8 latents, fp32, the two layers kept apart (no nonlinearity between them).  W2 must be
 * 16-byte aligned (AVC_E_ALIGN) and H a multiple of 4; workspace avc_vae_decode_workspace_bytes(B, H).
 * avc_load_textures is neural_renderer's load_textures (nr.load_obj(..., load_texture=True, texture_size=8),
 * utils.py:7) for ONE material image: image [height][width][3] float in [0, 1] as stored (row 0 = top; the vertical
 * flip of load_obj happens inside), face_uv [F][3][2] (the UV triangle of every face, any real value: REPEAT wraps
 * it into [0, 1)), is_update [F] (non-zero: the face uses this material), textures [F][R][R][R][3] updated in place
 * for those faces only (the caller fills it with 1.0 first, as load_obj does).  Texel (i, j, k) is the bilinear
 * sample at the barycentric point (i, j, k) / (i + j + k) of the UV triangle.  2 <= R <= 64.
 * avc_raster_textured is render_one_batch's render (utils.py:9-32, neural_renderer Renderer(camera_mode='look_at'):
 * 30 deg viewing angle, near 0.1, far 100, fill_back, black background) from eye / at / up (HOST pointers) of the
 * vertices as given: light 0.5 + 0.5 relu(n . (0, 1, 0)) per face with n = normalize((v0 - v1) x (v2 - v1)) facing
 * the eye, times the trilinear sample of the face's cube at the perspective-corrected barycentrics w_k (R - 1) z / z_k
 * clamped to [0, R - 1 - 1e-5], then the supersample x supersample average.  rgb_out [n][n][3], row 0 at the top
 * (neural_renderer's [3][n][n] image transposed to HWC).  Workspace: avc_raster_textured_workspace_bytes.
 * AVC_E_BADCFG when eye == at or up is parallel to the viewing direction.
 * avc_clip_prep_nearest: images [B][n][n][3] -> out [B][3][S][S], F.interpolate(size=S) (nearest: src =
 * floor(dst * n / S)) then the CLIP Normalize (main.py:101-103).
 * avc_codebook_argmax: cos_out[N] = F.normalize(codebook[N][D] - image_emb[D], dim=1) . F.normalize(delta[D])
 * (main.py:106-107, norms clamped at 1e-12) and best_out (device int32) = its first argmax (main.py:108); the
 * workspace holds at least 8 bytes.
 * ------------------------------------------------------------------------------------------ */
int avc_vae_decode_workspace_bytes(int32_t B, int32_t hidden, size_t* bytes);
int avc_vae_decode(const float* z, int32_t B, int32_t latent, const float* W1, const float* b1, int32_t hidden,
                   const float* W2, const float* b2, const float* v_template, int32_t out_dim, float* out,
                   void* workspace, size_t workspace_bytes, avc_stream_t stream);
int avc_load_textures(const float* image, int32_t height, int32_t width, const float* face_uv,
                      const int32_t* is_update, int32_t F, int32_t R, float* textures, avc_stream_t stream);
int avc_raster_textured_workspace_bytes(int32_t V, int32_t image_size, int32_t supersample, size_t* bytes);
int avc_raster_textured(const float* verts, const int32_t* faces, const float* textures, int32_t V, int32_t F,
                        int32_t R, const float* eye, const float* at, const float* up, int32_t image_size,
                        int32_t supersample, float* rgb_out, void* workspace, size_t workspace_bytes,
                        avc_stream_t stream);
int avc_clip_prep_nearest(const float* images, int32_t B, int32_t n, int32_t out_size, float* out,
                          avc_stream_t stream);
int avc_codebook_argmax(const float* codebook, const float* image_emb, const float* delta, int32_t N, int32_t D,
                        float* cos_out, int32_t* best_out, void* workspace, size_t workspace_bytes,
                        avc_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Video frames of a generated avatar (avatarclip_b200/video.py): one vertex-coloured mesh, smooth-shaded, over many
 * frames per launch.  The reference has no renderer for its results (render_novel_image / interpolate_view cannot
 * run, AvatarAnimate's visualize.py draws the grey SMPL body through pyrender); this one is the project's own.
 *
 * avc_video_adjacency: the vertex -> incident-face lists of faces [F][3] as CSR, built once per mesh: offsets [V + 1]
 * (offsets[V] = the number of entries, at most 3F), vf [3F] the face ids of vertex v in vf[offsets[v] .. offsets[v+1]),
 * in ascending face order (a face naming v twice is listed twice; an index outside [0, V) is skipped).
 * 1 <= V, 1 <= F <= 2^29.  Workspace: avc_video_adjacency_workspace_bytes(V).
 *
 * avc_video_render: rgb_out [n_frames][n][n][3] uint8 (n = image_size, row 0 at the top) of the mesh with vertices
 * verts + f * frame_stride ([V][3] per frame; frame_stride 0: every frame draws the same vertices).
 *   - cameras: HOST [n_frames][13]: a world-to-camera [R | t] (row-major 3x4; camera x right, y down, z forward), then
 *     the focal length in output pixels; the principal point is the image centre.  Each output pixel holds
 *     supersample x supersample samples at the centres of its sub-pixels.
 *   - Faces with a vertex at camera depth z <= 0.01 are skipped, both windings are drawn, and per sample the face of
 *     the smallest perspective-correct depth wins (64-bit atomicMin of (depth bits | face id): ties to the smaller id).
 *   - Vertex normal: the sum over the vertex's faces, in CSR order, of the un-normalised (v1 - v0) x (v2 - v0), per
 *     frame (no float atomics: the frames are bitwise reproducible).
 *   - Sample colour: the perspective-correct barycentric interpolation of the stored 0-255 colours (colors [V][3]
 *     uint8, or NULL for a uniform grey of 200) times 0.25 + 0.75 max(0, n . v), n the interpolated normal,
 *     normalised and flipped to face the camera, v the direction towards the camera along its axis (a headlight);
 *     background (HOST [3] uint8) where no face won.  The pixel is the mean of its samples rounded to nearest.
 *   - face_out: NULL, or [n_frames][n * supersample][n * supersample] int32, the winning face of every sample (-1:
 *     none), row 0 at the top.
 *   - AVC_E_BADCFG unless 1 <= image_size <= 4096, 1 <= supersample <= 4, 1 <= n_frames <= 65535, V >= 1,
 *     1 <= F <= 2^29, frame_stride >= 0 and every focal length > 0.
 *   - offsets / vf from avc_video_adjacency of the same faces.  Workspace: avc_video_render_workspace_bytes (about
 *     n_frames * (32 V + 8 (n * supersample)^2) bytes).
 * ------------------------------------------------------------------------------------------ */
int avc_video_adjacency_workspace_bytes(int32_t V, size_t* bytes);
int avc_video_adjacency(const int32_t* faces, int32_t V, int32_t F, int32_t* offsets, int32_t* vf, void* workspace,
                        size_t workspace_bytes, avc_stream_t stream);
int avc_video_render_workspace_bytes(int32_t V, int32_t F, int32_t n_frames, int32_t image_size, int32_t supersample,
                                     size_t* bytes);
int avc_video_render(const float* verts, int64_t frame_stride, const int32_t* faces, const int32_t* offsets,
                     const int32_t* vf, const uint8_t* colors, int32_t V, int32_t F, const float* cameras,
                     int32_t n_frames, int32_t image_size, int32_t supersample, const uint8_t* background,
                     uint8_t* rgb_out, int32_t* face_out, void* workspace, size_t workspace_bytes,
                     avc_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* AVC_B200_H */
