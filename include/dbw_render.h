/*
 * include/dbw_render.h -- C-ABI of the H100-native (sm_90a) differentiable primitive renderer.
 *
 * The reference (monniert/differentiable-blocksworld) has no FFI: its render hot path is a Python-level seam,
 *     Renderer.forward(meshes, R, T, viz_purpose=False, **kwargs) -> (B,4,H,W)      src/model/renderer.py:84-98
 * behind which PyTorch3D's MeshRasterizer (_C.rasterize_meshes / _C.rasterize_meshes_backward) and the
 * reference's LayeredShader + layered_rgb_blend (src/model/renderer.py:219-273) run.  This header is what a
 * binding for that seam loads instead: plain pointers and sizes, no torch types.  Each entry point cites the
 * reference interface it replaces.  INTEGRATION.md shows the ctypes stub on the reference side.
 *
 * Conventions
 *  - every pointer except `settings` is a DEVICE pointer on the current CUDA device (the *_host entry points
 *    take HOST pointers and do the copies themselves);
 *  - the caller owns every buffer; the library never allocates or frees device memory (the *_host entry
 *    points keep one grow-only per-process scratch arena, released by dbw_host_arena_release());
 *  - all work is ordered on `stream` (a cudaStream_t passed as void*); no implicit synchronisation;
 *  - gradient outputs ACCUMULATE (atomics): the caller zero-fills them;
 *  - return value 0 = success, negative = error (message via dbw_last_error(), thread-local); never throws;
 *  - dtype is float32 throughout; ids are int32.
 */
#ifndef DBW_RENDER_H
#define DBW_RENDER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DBW_ABI_VERSION 8
#define DBW_MAX_FACES_PER_PIXEL 64

/*
 * Mirrors RasterizationSettings + BlendParams + the LayeredShader flags the reference configures at
 * src/model/renderer.py:29-54 and the camera it installs at src/model/dbw.py:204-208.
 */
typedef struct DbwRenderSettings {
  int32_t n_views;            /* B: cameras / images in this call (Meshes.extend(B), src/model/dbw.py:215,220)      */
  int32_t height, width;      /* img_size (H, W)                                                                    */
  int32_t faces_per_pixel;    /* K  (renderer.py:33)                                                                */
  int32_t n_verts, n_faces;   /* V, F of the (single) scene mesh shared by all views                                 */
  int32_t n_maps;             /* M texture maps (join_meshes_as_scene keeps one per sub-mesh)                        */
  int32_t alpha_view_stride;  /* faces_alpha layout: 0 = (F,) shared by all views; F = (B*F,) batch-packed (dbw.py:219) */
  float fx, fy, px, py;       /* PerspectiveCameras K in NDC (src/dataset/dtu.py:102-106): K[0,0], K[1,1], K[0,2], K[1,2] */
  float sigma;                /* BlendParams.sigma (renderer.py:31); 0 = hard                                        */
  float blur_radius;          /* log(1/1e-4 - 1) * sigma (renderer.py:51)                                            */
  float z_clip;               /* z_clip_value (renderer.py:35,46); < 0 disables clipping                             */
  float proj_eps;             /* eps passed to the cameras (renderer.py:20,94) = 1e-8                                 */
  float background[3];        /* BlendParams.background_color (renderer.py:32)                                       */
  int32_t clip_inside;        /* LayeredShader clip_inside (renderer.py:41)                                          */
  int32_t perspective_correct;/* renderer.py:34,46 (None -> True for perspective cameras)                            */
  int32_t clip_barycentric;   /* clip_barycentric_coords=True (renderer.py:46)                                       */
  int32_t detach_bary;        /* LayeredShader detach_bary (renderer.py:43,222-223): no gradient through barycentrics */
  int32_t verts_are_ndc;      /* 1: `verts` is (B,V,3) = (x_ndc, y_ndc, z_view) and R/T/K are ignored                 */
  int32_t n_map_floats;       /* total floats in `maps` (= 3 * sum_m H_m*W_m): sizes the library's float4 texel scratch    */
  int32_t maps_are_texels4;   /* 1: `maps` (and `g_maps`) are already RGB+pad float4 texel atlases (dbw_texture_prep_*);
                                 DbwMapDesc.offset keeps its meaning (3 * first texel index).  2: the same, and the table
                                 holds cell maps (DBW_MAP_CELLS): the backward spreads their gradient atomics over
                                 DBW_CELL_GRAD_COPIES copies in its scratch and adds the copies into g_maps at the end (a
                                 cell collects the gradient of f x f texels: one copy would serialise the atomics of
                                 every warp that covers it)                                                               */
  int32_t save_fragment_state;/* 1: the forward also keeps one 16 B record {triangle slot | closest edge, u, v, signed squared
                                 distance} and one 16 B colour {r, g, b, -} per kept fragment (+ a per-pixel count byte) in its
                                 workspace; dbw_render_backward streams these instead of re-deriving geometry and REQUIRES
                                 them.  Costs B*H*W*(32 K + 1) bytes of workspace ADDRESS space (only fragments that exist are
                                 touched).  2: the same for a pass without opacities (faces_alpha must then be NULL in the
                                 forward and the backward); when it is also hard and single-layer (sigma = 0, K = 1) its
                                 backward has no use for the colours and they are not kept: B*H*W*(16 + 1) bytes            */
  int32_t alpha_group;        /* faces sharing one opacity entry (0/1: one per face).  faces_alpha / g_faces_alpha then have
                                 n_faces / alpha_group entries per view: a DBW block is 80 faces with ONE opacity
                                 (src/model/dbw.py:219 repeat_interleave's it per face; that is alpha_group = 1)            */
  int32_t n_static_faces;     /* faces [0, n_static_faces) have constant vertices (the background sphere of the environment,
                                 src/model/dbw.py:267-280): the backward skips their vertex gradient.  Ignored (0) by a
                                 dbw_render_backward call that asks for camera gradients                                    */
  const int32_t* view_rows;   /* DEVICE (B,2) int32 or NULL: [row_begin, row_end) of each view that this call renders / differentiates.
                                 Rows outside are left untouched in every output (and contribute nothing to a fused loss):
                                 a data-parallel step shards at (view, row band) granularity, so 49 views split evenly
                                 over 8 ranks (SURVEY 8e)                                                                   */
} DbwRenderSettings;

/* Texture table entry: map m lives at maps[offset .. offset + height*width*3), row-major (H, W, 3).
 * reserved = 0: that layout.  reserved = DBW_MAP_CELLS(f, p_left): a CELL map -- an f x f box-decimated square texture
 * (DBW_TEX_STAGE_CELLS4 output, maps_are_texels4 = 2) stored as its (height/f) x (height/f) cells, row-major, one float4 per
 * cell, from cell offset / 3 on.  height and width still describe the logical atlas the cells stand for (TS rows,
 * p_left + TS + p_right columns of circular padding along u, as DBW_TEX_STAGE_EXPAND would write it), so sampling is
 * unchanged: every bilinear tap reads (and its gradient goes to) the cell its atlas texel would repeat.  Renders are bit
 * for bit those of the expanded atlas; texture gradients are the atlas gradients summed per cell (what
 * DBW_TEX_STAGE_EXPAND's backward computes), up to summation order.  The caller keeps offset / 3 + (height/f)^2 within the
 * n_map_floats / 3 cells of `maps`.  f is a power of two in [2, 128], height % f == 0, 0 <= p_left <= height. */
typedef struct DbwMapDesc { int32_t offset, height, width, reserved; } DbwMapDesc;
#define DBW_MAP_CELLS(f, p_left) (((p_left) << 8) | (f))
#define DBW_CELL_GRAD_COPIES 8

int dbw_abi_version(void);
/* Test hook: 1 = hard single-layer renders (K = 1, sigma = 0) go through the generic raster kernel instead of their dedicated one. */
void dbw_debug_generic_kernel_only(int on);
/* Test hook: 1 = keep writing what no backward reads (the colours of a save_fragment_state = 2 hard single-layer pass, the
 * alpha plane of an env_alpha_unread epilogue's g_env), for tests that compare against the computation that writes them.  Set it before
 * dbw_workspace_bytes: it changes the forward workspace's size. */
void dbw_debug_keep_unread_outputs(int on);
/* sizeof(DbwRenderSettings) as compiled into the library: lets a binding verify its mirror of the struct. */
size_t dbw_sizeof_settings(void);
const char* dbw_last_error(void);

/* Bytes of the two caller-provided device scratch buffers:
 *   *fwd_bytes: workspace written by dbw_render_forward and read again by dbw_render_backward (keep it alive);
 *   *bwd_bytes: scratch used only inside dbw_render_backward. */
int dbw_workspace_bytes(const DbwRenderSettings* settings, size_t* fwd_bytes, size_t* bwd_bytes);

/*
 * Forward of Renderer.forward (src/model/renderer.py:84-98): projection -> z-clip -> rasterize (top-K nearest
 * faces per pixel within the blur halo) -> UV interpolation + bilinear texture fetch -> layered soft blend.
 *   verts        (V,3) world-space vertices   [or (B,V,3) NDC when settings->verts_are_ndc]
 *   faces        (F,3) int32 vertex ids
 *   faces_uvs    (F,3,2) per-face-vertex UVs = verts_uvs[faces_uvs] of TexturesUV (src/model/dbw.py:280,295,342)
 *   face_map     (F) int32 texture map of each face; a NEGATIVE entry disables the face (it is never rasterized and gets
 *                no gradient) -- how a static-topology caller drops low-opacity blocks (src/model/dbw.py:316-328)
 *   maps, map_table  packed maps + (M) DbwMapDesc (device)
 *   R (B,3,3), T (B,3)  row-vector convention X_view = X_world @ R + T (src/dataset/dtu.py:75-124)
 *   faces_alpha  NULL, or per-face opacity (src/model/dbw.py:219, renderer.py:258-260), see alpha_view_stride / alpha_group
 *   out_rgba     (B,4,H,W)  RGB + coverage, NCHW (renderer.py:268)
 *   topk_ids     (B,K,H,W) int32 or NULL: z-sorted face slots kept per pixel (-1 = empty) = fragments.pix_to_face modulo
 *                the slot convention; a diagnostic / visualisation output (render_edges), NOT what the backward reads --
 *                that is the workspace's fragment records (settings->save_fragment_state)
 * and the two optional extras the reference's visualisation paths need (SURVEY 8f ranks 2 and 4):
 *   face_shade   (B,F,3) or NULL: per-view per-face colour multiplier = PyTorch3D flat shading with ambient + directional
 *                diffuse light, as configured for renderer_light (src/model/dbw.py:139-143, renderer.py:87-97,195-205)
 *   out_dists    (B,K,H,W) or NULL: signed squared NDC distance of each kept fragment to its face's nearest edge
 *                (< 0 inside, -1 for empty slots) = fragments.dists, what render_edges thresholds (renderer.py:134-146)
 */
int dbw_render_forward(const DbwRenderSettings* settings, const float* verts, const int32_t* faces,
                       const float* faces_uvs, const int32_t* face_map, const float* maps,
                       const DbwMapDesc* map_table, const float* R, const float* T, const float* faces_alpha,
                       float* out_rgba, int32_t* topk_ids, void* workspace, size_t workspace_bytes,
                       const float* face_shade, float* out_dists, void* stream);

/*
 * Backward of the same (replaces autograd through layered_rgb_blend, grid_sample, interpolate_face_attributes
 * and _C.rasterize_meshes_backward).  grad_rgba (B,4,H,W), multiplied by the device scalar *grad_scale (NULL = 1) as it is
 * read.  Outputs accumulate:
 *   g_verts        (V,3)  [or (B,V,3) when verts_are_ndc]
 *   g_faces_alpha  same shape as faces_alpha (may be NULL when faces_alpha is NULL)
 *   g_maps         same packing as maps (may be NULL: no texture gradient)
 * and the gradient of the camera poses (PyTorch3D keeps the camera transform inside autograd behind the reference's
 * renderer, src/model/renderer.py:94, so a loss on the image differentiates R and T):
 *   g_R (B,3,3), g_T (B,3)  accumulate (the caller zero-fills); either may be NULL.  Row-vector convention
 *                           X_view = X_world @ R + T:  g_T[b] = sum_v g_view[b,v],  g_R[b][i][j] = sum_v X_world[v][i] g_view[b,v][j],
 *                           g_view the NDC vertex gradient pulled back through the projection (|z| < proj_eps: no z term).
 * Requires the forward to have run with save_fragment_state = 1 or 2 on the same workspace.  With g_R or g_T set:
 *  - n_static_faces is treated as 0: every face moves in the image when the camera does, so the static faces are
 *    differentiated too (the background sphere of the environment pass), and g_verts, when not NULL, then also receives the
 *    rows of the static faces' vertices;
 *  - the per-view sums run in a fixed order (one CTA per view) and each element of g_R / g_T receives one atomic add per call;
 *  - with view_rows, the result is the gradient of the rows this call owns: the calls over a partition of the rows sum to
 *    the gradient of the whole image;
 *  - verts_are_ndc is an error (R and T are not part of such a render).
 */
int dbw_render_backward(const DbwRenderSettings* settings, const float* verts, const int32_t* faces,
                        const float* faces_uvs, const int32_t* face_map, const float* maps,
                        const DbwMapDesc* map_table, const float* R, const float* T, const float* faces_alpha,
                        const void* workspace, size_t workspace_bytes, const float* grad_rgba, const float* grad_scale,
                        float* g_verts, float* g_faces_alpha, float* g_maps, float* g_R, float* g_T,
                        void* bwd_scratch, size_t bwd_scratch_bytes, void* stream);

/*
 * Fused compositing + RGB loss of the decoupled scene (src/model/dbw.py:223 and :366-367):
 *   rec = rgb_fg * a_fg + (1 - a_fg) * rgb_env ;  loss = weight * mean((imgs - rec)^2)
 * fg, env: (B,4,H,W) outputs of dbw_render_forward; imgs (B,3,H,W).  Writes rec (B,3,H,W) (may be NULL), adds
 * the loss into *loss_sum (device scalar, caller zero-fills), and -- when g_fg / g_env are not NULL -- writes the
 * gradients of `loss` w.r.t. fg and env ((B,4,H,W), overwritten).  `inv_count` = weight / (B_total*3*H*W).
 */
int dbw_composite_mse(int32_t n_views, int32_t height, int32_t width, const float* fg, const float* env,
                      const float* imgs, float inv_count, float* rec, float* loss_sum, float* g_fg, float* g_env,
                      void* stream);

/* Backward of dbw_composite_mse: d(g_loss * loss + <g_rec, rec>) / d fg, d env, written to g_fg / g_env ((B,4,H,W)).
 * g_loss: device scalar (may be NULL = 0); g_rec: (B,3,H,W) gradient arriving at `rec` from other losses (may be NULL). */
int dbw_composite_mse_backward(int32_t n_views, int32_t height, int32_t width, const float* fg, const float* env,
                               const float* imgs, float inv_count, const float* g_loss, const float* g_rec, float* g_fg,
                               float* g_env, void* stream);

/*
 * Fused loss epilogue (SURVEY 8f rank 3: "MSE fused into blend").  dbw_render_forward_loss is dbw_render_forward for the
 * LAST layer of a decoupled render (the blocks, src/model/dbw.py:219-223) with the compositing over the already rendered
 * environment and the RGB loss (dbw.py:366-367, nn.MSELoss) done in the rasterizer's epilogue, per pixel, while the blended
 * colour is still in registers:
 *     rec = rgb * a + (1 - a) * rgb_env ;  loss = sum((rec - target)^2) * inv_count
 * Instead of the image, `out_rgba` receives d loss / d (this layer's RGBA) and `g_env` d loss / d env_rgba (alpha plane 0, or unwritten: env_alpha_unread),
 * i.e. exactly the grad_rgba inputs of the two dbw_render_backward calls (scaled there by the upstream gradient of the
 * loss through `grad_scale`): no composite kernel, no image round trip through HBM in either direction.
 */
typedef struct DbwLossEpilogue {
  const float* env_rgba;      /* (B,4,H,W) render of the layer behind (dbw_render_forward output)                          */
  const float* target;        /* (B,3,H,W) ground-truth images                                                             */
  float* g_env;               /* (B,4,H,W) out: d loss / d env_rgba                                                        */
  float* rec;                 /* (B,3,H,W) out: composited image, or NULL                                                  */
  float* loss_partials;       /* (n_partials) out: zero-filled by the call, then partial sums; loss = their sum            */
  int32_t n_partials;         /* power of two, >= 1                                                                        */
  float inv_count;            /* weight / (B_total * 3 * H * W): the mean of nn.MSELoss over the GLOBAL batch              */
  int32_t env_alpha_unread;   /* 1: nothing reads the alpha plane of g_env and it is left unwritten -- the environment's
                                 backward has no opacity and no distance path (sigma = 0, faces_alpha NULL), and such a
                                 dbw_render_backward never reads grad_rgba's alpha plane.  0: the plane is written (zeros)  */
} DbwLossEpilogue;

int dbw_render_forward_loss(const DbwRenderSettings* settings, const float* verts, const int32_t* faces,
                            const float* faces_uvs, const int32_t* face_map, const float* maps,
                            const DbwMapDesc* map_table, const float* R, const float* T, const float* faces_alpha,
                            float* out_g_rgba, int32_t* topk_ids, void* workspace, size_t workspace_bytes,
                            const DbwLossEpilogue* epilogue, void* stream);

/*
 * dbw_render_forward_loss for a detach_bary pass over float4 cell maps (maps_are_texels4 = 2) that also runs the pass's
 * backward inside the same kernel, on the per-pixel fragment lists while they are still on chip: the texture scatter, the
 * opacity sums and the distance-path vertex gradients go, unscaled, into `bwd_scratch` (dbw_workspace_bytes' bwd size; the
 * call zero-fills it), and dbw_render_backward_deferred later folds them into the caller's gradients, multiplied by the
 * upstream gradient of the loss.  No fragment records are written (save_fragment_state must be 0) and no d loss / d RGBA
 * image either; g_env is written as by dbw_render_forward_loss.  grad_mask: which gradients the later fold will ask for
 * (DBW_GRAD_VERTS also for camera gradients).  The loss terms are those of dbw_render_forward_loss, bit for bit.
 */
#define DBW_GRAD_VERTS 1
#define DBW_GRAD_MAPS 2
#define DBW_GRAD_ALPHA 4
int dbw_render_forward_loss_grad(const DbwRenderSettings* settings, const float* verts, const int32_t* faces,
                                 const float* faces_uvs, const int32_t* face_map, const float* maps,
                                 const DbwMapDesc* map_table, const float* R, const float* T, const float* faces_alpha,
                                 void* workspace, size_t workspace_bytes, const DbwLossEpilogue* epilogue, int32_t grad_mask,
                                 void* bwd_scratch, size_t bwd_scratch_bytes, void* stream);

/*
 * The rest of the backward of a dbw_render_forward_loss_grad call (same settings, workspace and scratch): adds
 * *grad_scale (device scalar, required) times the scratch into g_maps (the cell-gradient copies), g_faces_alpha and, through
 * the face setup and projection backward, g_verts, g_R and g_T (any may be NULL; camera gradients as in
 * dbw_render_backward).  A gradient whose grad_mask bit the forward did not set comes out unchanged.
 */
int dbw_render_backward_deferred(const DbwRenderSettings* settings, const float* verts, const int32_t* faces, const float* R,
                                 const float* T, const void* workspace, size_t workspace_bytes, const float* grad_scale,
                                 float* g_verts, float* g_faces_alpha, float* g_maps, float* g_R, float* g_T,
                                 void* bwd_scratch, size_t bwd_scratch_bytes, void* stream);

/*
 * Fused scene construction (src/model/dbw.py:267-352), so that a training step needs no eager tensor ops between the
 * leaf parameters and the rasterizer.  All pointers are device pointers.
 */
typedef struct DbwSceneGeometry {
  int32_t n_blocks, verts_per_block, n_ground_verts, reserved;
  const float* sq_eta;        /* (N,Vb) buffers sq_eta / sq_omega (dbw.py:86-87)                                           */
  const float* sq_omega;
  const float* sq_eps;        /* (N,2)  dbw.py:84, eps = sigmoid(.)*1.8 + 0.1 (dbw.py:349)                                 */
  const float* S;             /* (N,3)  scale = exp(S) + scale_min (dbw.py:299)                                            */
  const float* R_6d;          /* (N,6)  rotation_6d_to_matrix (dbw.py:299)                                                 */
  const float* T;             /* (N,3)                                                                                     */
  const float* ground_verts;  /* (Vg,3) static plane vertices (dbw.py:76-78); may be NULL when n_ground_verts == 0         */
  const float* R_6d_ground;   /* (6)    dbw.py:99,285                                                                      */
  const float* T_ground;      /* (3)    dbw.py:100                                                                         */
  float ratio_block_scene, scale_min, S_world;
  float R_world[9], T_world[3];   /* world transform (v * S_world) @ R_world + T_world (dbw.py:264,344)                    */
} DbwSceneGeometry;

/* World-space vertices of the N superquadric blocks and of the ground plane, in the layout the two render passes consume
 * without a concatenation: verts_out (n_env_static + Vg + N*Vb, 3) = the static environment vertices (the background sphere
 * in world space, dbw.py:271-274; copied; there may be none), the ground, then the blocks -- the environment pass takes the
 * first n_env_static + Vg rows, the blocks pass the rest.  The backward takes the two gradient blocks where they lie (any
 * two device pointers: no gather; each may be NULL when it has no rows) and writes the gradients of the leaf parameters
 * (written, not accumulated). */
int dbw_scene_geometry_forward(const DbwSceneGeometry* g, const float* env_static_verts, int32_t n_env_static,
                               float* verts_out, void* stream);
int dbw_scene_geometry_backward(const DbwSceneGeometry* g, const float* g_block_verts, const float* g_ground_verts,
                                float* g_sq_eps, float* g_S, float* g_R_6d, float* g_T, float* g_R_6d_ground,
                                float* g_T_ground, void* stream);

/* Block opacities of a step (src/model/dbw.py:300-316 with static shapes), one launch each way:
 *   alpha[k]      = sigmoid(alpha_logit[k] + noise_scale * noise[k])      (noise may be NULL)
 *   keep[k]       = keep_threshold < 0  ||  sigmoid(alpha_logit[k]) > keep_threshold      (0.5: hard filter, 0.01: kill_blocks)
 *   alpha_kept[k] = keep[k] ? alpha[k] : 0                                (optional)
 *   face_map_out[k*faces_per_block + j] = keep[k] ? face_map_in[..] : -1  (optional; -1 = never rasterized)
 * backward: g_alpha_logit = (g_alpha + keep * g_alpha_kept) * alpha * (1 - alpha)   (either gradient may be NULL). */
int dbw_opacity_forward(const float* alpha_logit, const float* noise, float noise_scale, float keep_threshold,
                        const int32_t* face_map_in, int32_t n_blocks, int32_t faces_per_block, float* alpha, float* alpha_kept,
                        int32_t* face_map_out, void* stream);
int dbw_opacity_backward(const float* alpha_logit, const float* noise, float noise_scale, float keep_threshold,
                         const float* g_alpha, const float* g_alpha_kept, int32_t n_blocks, float* g_alpha_logit, void* stream);

/* textures (M,TS,TS,3) logits -> atlas (M, TS, p_left+TS+p_right) float4 texels: sigmoid, optional `decimate`xdecimate box
 * filter (1 = off, 8 = dbw.py:331-334), circular padding along u (dbw.py:339-341).  Backward: g_atlas -> g_textures. */
/* One texture stack of a multi-stack texture preparation: (n_maps, txt_size, txt_size, 3) logits -> float4 texel atlas
 * (n_maps, txt_size, p_left + txt_size + p_right) [forward: `atlas` is written; backward: `atlas` is the atlas GRADIENT that is read
 * and `g_textures` receives d/d logits]. */
/* `stage` splits the preparation at the CELL COLOURS c = box_mean(sigmoid(logits)), (n_maps, txt_size/decimate, txt_size/decimate, 3)
 * floats -- the smallest tensor on the way (64x smaller than the textures while they are decimated), where a data-parallel
 * trainer sums gradients over ranks (parallel.GradSumPoint):
 *   DBW_TEX_STAGE_FUSED   logits -> atlas                                     (backward: atlas gradient -> logit gradient)
 *   DBW_TEX_STAGE_CELLS   logits -> cells, written to `atlas`                 (backward: `atlas` = CELL gradient -> logit gradient)
 *   DBW_TEX_STAGE_EXPAND  cells (passed as `textures`) -> atlas               (backward: atlas gradient -> cell gradient, written
 *                                                                              to `g_textures`; `textures` is not read)
 *   DBW_TEX_STAGE_CELLS4  as CELLS, but the cells are float4 (RGB + 0, 16-byte aligned): the maps of DBW_MAP_CELLS map
 *                         table entries, which the raster kernels sample without an atlas (backward: `atlas` = float4 cell
 *                         gradient, read with 4-byte loads -> logit gradient)
 * CELLS then EXPAND equals FUSED bit for bit, forward and backward. */
#define DBW_MAX_TEX_JOBS 4
#define DBW_TEX_STAGE_FUSED 0
#define DBW_TEX_STAGE_CELLS 1
#define DBW_TEX_STAGE_EXPAND 2
#define DBW_TEX_STAGE_CELLS4 3
typedef struct DbwTexJob {
  const float* textures; float* atlas; float* g_textures;
  int32_t n_maps, txt_size, p_left, p_right, decimate, stage;
} DbwTexJob;
/* Several stacks in ONE launch (the step's three: background, ground, blocks; `jobs` is a HOST array of n_jobs <= 4). */
int dbw_texture_prep_forward_multi(const DbwTexJob* jobs, int32_t n_jobs, void* stream);
int dbw_texture_prep_backward_multi(const DbwTexJob* jobs, int32_t n_jobs, void* stream);

/*
 * Host-buffer variants (the end-to-end call a reference-side binding makes with numpy / CPU tensors): every
 * pointer is a HOST pointer; the library stages through its own device arena on the current device, runs the
 * device entry points above on `stream`, copies results back and synchronises the stream before returning.
 */
int dbw_render_forward_host(const DbwRenderSettings* settings, const float* verts, const int32_t* faces,
                            const float* faces_uvs, const int32_t* face_map, const float* maps, size_t maps_floats,
                            const DbwMapDesc* map_table, const float* R, const float* T, const float* faces_alpha,
                            float* out_rgba, void* stream);
void dbw_host_arena_release(void);

/* Number of kernel launches issued by this library since process start (for bench.py's gpu_launches). */
uint64_t dbw_launch_count(void);

/* Optional live timing of the two rasterization kernels with CUDA events on the launch stream (bench.py's roofline):
 * kind 0 = raster forward, 1 = raster backward; K filters by faces_per_pixel (0 = any).  dbw_timing_read synchronises
 * on the recorded events and returns their summed duration and count; dbw_timing_reset frees them. */
void dbw_timing_enable(int on);
int dbw_timing_read(int kind, int K, double* total_ms, int* count);
void dbw_timing_reset(void);

/*
 * The step's one gradient exchange (SURVEY 8e: views shard with no data-path collective; ONE all-reduce(SUM) of the flat
 * parameter-gradient bucket) as a hand-written all-reduce over NVLink peer memory -- a plain kernel launch on `stream`,
 * hence capturable inside the step's CUDA graph.  One process per GPU of one node:
 *   dbw_comm_create      allocates this rank's arena (bucket of max_floats + inbox of the same size + control; cudaMalloc)
 *   dbw_comm_buffer      the arena's bucket: the caller keeps its gradients THERE (nothing is staged or copied)
 *   dbw_comm_ipc_handle  64-byte cudaIpcMemHandle of the arena, to be all-gathered by the caller (torch.distributed)
 *   dbw_comm_connect     opens the peers' arenas: all_handles = world x 64 bytes in rank order
 *   dbw_comm_all_reduce  in-place SUM of the bucket's first n_floats over the ranks (n_floats % 4 == 0; buf must be the
 *                        pointer dbw_comm_buffer returned).  Push protocol: slices are pushed to their owners, summed there
 *                        in rank order (bit-identical results everywhere) and pushed back -- only posted stores cross NVLink
 *   dbw_comm_error       0, or which barrier timed out (a peer did not arrive within ~30 s: results are garbage, no hang)
 */
int dbw_comm_create(int32_t world, int32_t rank, size_t max_floats, void** comm_out);
int dbw_comm_buffer(void* comm, float** out);
int dbw_comm_ipc_handle(void* comm, void* out_handle64);
int dbw_comm_connect(void* comm, const void* all_handles);
int dbw_comm_all_reduce(void* comm, float* buf, size_t n_floats, void* stream);
int dbw_comm_error(void* comm, int32_t* out);
int dbw_comm_destroy(void* comm);

/*
 * DTU chamfer evaluation (the reference's utils/dtu_eval.evaluate_mesh, run at the end of Trainer.evaluate() on a DTU
 * scene): mesh point sampling, greedy radius downsampling and exact nearest-neighbour distances, all in fp64 with
 * non-contracting arithmetic (bit-identical samples, distances sqrt((dx^2 + dy^2) + dz^2)).  Points are (N,3) double.
 * The entry points are the per-point stages; scans and sorts between them are the caller's (dbw_b200/dtu_eval.py
 * uses torch.cumsum / torch.sort).  Same conventions as above: device pointers, caller-owned buffers, `stream`, 0 = ok.
 *
 * Uniform grid of cells of edge `cell` from `origin`; dims are cell counts per axis.  block = 1: a point's key is its
 * linear cell (x + nx * (y + ny * z)).  block = B > 1 (dims multiples of B): block-major keys, so that the B^3 cells of one
 * block are consecutive and a block's occupancy is the difference of two cell offsets.  Cell coordinates are clamped into
 * the grid.
 */
typedef struct DbwEvalGrid {
  double origin[3];
  double cell;
  int64_t dims[3];
  int32_t block, reserved;
} DbwEvalGrid;

/* Sampling, pass 1 (per triangle): tri (F,12) records (t0, v1, v2, n1, n2, -) and n_rows (F): the lattice rows of each
 * triangle (0 for zero-area triangles and triangles with n1 == 0 or n2 == 0).  faces (F,3) int64 index verts (V,3). */
int dbw_eval_sample_setup(const double* verts, const int64_t* faces, int64_t n_faces, double* tri, int64_t* n_rows, void* stream);
/* Pass 2 (per row): row_begin (F+1) = exclusive scan of n_rows; row_count (n_rows_total) = samples of each row. */
int dbw_eval_sample_count(const double* tri, const int64_t* row_begin, int64_t n_faces, int64_t n_rows_total,
                          int64_t* row_count, void* stream);
/* Pass 3 (one warp per row): sample_begin (n_rows_total) = exclusive scan of row_count; out (S,3) receives the samples
 * in the reference's order (triangle, then row-major over (i, j)). */
int dbw_eval_sample_write(const double* tri, const int64_t* row_begin, int64_t n_faces, int64_t n_rows_total,
                          const int64_t* row_count, const int64_t* sample_begin, double* out, void* stream);

/* keys (N) int64 of points (N,3) on `grid` (a HOST pointer). */
int dbw_eval_cell_keys(const double* points, int64_t n, const DbwEvalGrid* grid, int64_t* keys, void* stream);

/* Greedy radius downsample = the lexicographically-first maximal independent set of the graph dist <= radius, in ORDER
 * (a point's rank is its position in the shuffled cloud).  Inputs, on a block = 1 grid whose cell is >= radius:
 *   points   (N,3) sorted by cell key;  rank (N) int64 order position of each sorted point
 *   cell_of  (N) int32 index of each sorted point's cell in the C occupied cells
 *   nbr_begin, nbr_end (C,9) int32: sorted-point ranges of the 3x3x3 neighbourhood, one x-run per (dy, dz)
 *            (dbw_eval_cell_ranges)
 * Output keep (N) uint8 indexed by RANK.  Runs parallel rounds (keep a point once every earlier neighbour is removed,
 * remove it once one is kept) until every point is decided, reading a device counter after each round: this call
 * synchronises `stream`.  *rounds_out (host) = rounds run; more than max_rounds is an error, never a spin. */
int dbw_eval_cell_ranges(const int64_t* cell_keys, const int64_t* cell_begin, int64_t n_cells, const DbwEvalGrid* grid,
                         int32_t* nbr_begin, int32_t* nbr_end, void* stream);
int dbw_eval_downsample_workspace_bytes(int64_t n, size_t* bytes);
int dbw_eval_radius_downsample(const double* points, const int64_t* rank, const int32_t* cell_of, const int32_t* nbr_begin,
                               const int32_t* nbr_end, int64_t n, double radius, int32_t max_rounds, uint8_t* keep,
                               int32_t* rounds_out, void* workspace, size_t workspace_bytes, void* stream);

/* Exact 1-NN distance of each query to the targets, searched within max_dist: dist (n_queries) = the distance when one
 * is < max_dist, +inf otherwise.  targets (n_targets,3) sorted by block-major key on `grid` (block > 1);
 * cell_start (dims product + 1) int32 = first sorted target of each key.  The search walks rings of blocks around the
 * query, skips empty blocks and blocks farther than the best distance so far, and stops once the next ring cannot hold
 * anything closer.  Queries are best passed sorted by the same keys (coherent warps). */
int dbw_eval_nn_distance(const double* queries, int64_t n_queries, const double* targets, const int32_t* cell_start,
                         const DbwEvalGrid* grid, double max_dist, double* dist, void* stream);

/*
 * k-nearest neighbours (pytorch3d.ops.knn_points, D = 3, squared L2): the search under the reference's chamfer distance
 * (src/utils/chamfer.py), hence ChamferLoss, gradient_icp and the chamfer legs of ems_eval.py / mbf_eval.py.  Exact brute
 * force.  p1 (N,P1,3), p2 (N,P2,3) fp32; lengths1, lengths2 (N) int64 (clamped to [0, P]); N <= 65535, P < 2^31 - 1.
 *
 * dbw_knn_forward writes every element of dists (N,P1,K) fp32 and idx (N,P1,K) int64 (no zero-fill needed):
 *  - per query i < lengths1[n], the K nearest of p2[n, :lengths2[n]] in ascending (distance, index) order: ties go to
 *    the lower index;
 *  - distance = (dx*dx + dy*dy) + dz*dz, dx = p1.x - p2.x, each operation rounded to nearest fp32 (no contraction);
 *  - a target at a distance that is not below +inf (overflow, NaN) is never selected;
 *  - padding as PyTorch3D 0.7.1 (as recalled): rows i >= lengths1[n] and slots beyond the points found are dist 0, idx 0.
 * 1 <= K <= DBW_KNN_MAX_K.
 *
 * dbw_knn_backward: for i < lengths1[n] and k < min(K, lengths2[n]), with j = idx[n,i,k] (skipped outside
 * [0, lengths2[n])) and g = grad_dists[n,i,k]:  grad_p1[n,i] += 2 g (p1[n,i] - p2[n,j]),  grad_p2[n,j] -= the same
 * (fp32 atomics: the order of the additions into grad_p2 is not fixed).  The caller zero-fills both.
 */
#define DBW_KNN_MAX_K 32
int dbw_knn_forward(const float* p1, const float* p2, const int64_t* lengths1, const int64_t* lengths2, int64_t N, int64_t P1,
                    int64_t P2, int32_t K, float* dists, int64_t* idx, void* stream);
int dbw_knn_backward(const float* p1, const float* p2, const int64_t* lengths1, const int64_t* lengths2, const int64_t* idx,
                     const float* grad_dists, int64_t N, int64_t P1, int64_t P2, int32_t K, float* grad_p1, float* grad_p2,
                     void* stream);

/*
 * LPIPS (lpips 0.1.4, LPIPS(net='vgg', version='0.1'), as recalled): the perceptual term of the reference's objective.
 * in0 (imgs), in1 (rec): (B,3,H,W) fp32 NCHW, 16 <= H, W (relu5_3 is then at least 1x1), 1 <= B <= 65535,
 * B*H*W < 2^31 - 128.  value[b] = sum over the taps relu1_2 .. relu5_3 of the spatial mean of
 * lin_k . (dropout(n0 - n1)^2), n = f / (||f||_2 over channels + 1e-10).  With `normalize` the images are first mapped by
 * 2x - 1; then (x - shift) / scale.  The convolutions of 64..512 channels take TF32 operands (round to nearest, ties
 * away from zero) and accumulate in fp32; the first layer and its input-gradient are fp32.
 *
 * Dropout (p = 0.5, the reference's lin layers in training mode): with `train`, each (image, tap, channel, pixel) element
 * of the squared difference is kept and doubled when the hash of csrc/dbw_lpips_hash.cuh, for the seed *seed, says so,
 * and zeroed otherwise.  The forward copies *seed into the workspace for the backward and then increments *seed on the
 * device, so a captured graph draws a fresh mask on every replay.
 *
 * conv_w[l] (C_out, C_in, 3, 3) and conv_b[l] (C_out) of the 13 layers of torchvision's vgg16.features[0:30], lin_w[k]
 * (C_k) of the 5 heads, shift and scale (3): device fp32.  `prepared` (prepared_bytes from dbw_lpips_workspace_bytes)
 * holds the TF32-rounded forward copies [co][ky][kx][ci] and input-gradient copies [ci][2-ky][2-kx][co] of layers 1..12,
 * written by dbw_lpips_prepare_weights (again whenever the weights change).
 *
 * dbw_lpips_forward writes value (B).  With save_for_backward it keeps in the workspace what dbw_lpips_backward needs:
 * every activation of in1, the taps of in0, the seed used; without it, the workspace (sized with the same flag) holds
 * only the taps of both images.  dbw_lpips_backward writes grad_in1 (B,3,H,W) = sum_b grad_value[b] d value[b] / d in1
 * from the workspace of a save_for_backward forward (the same normalize and train; the workspace untouched in between).  Both run on `stream` only: no
 * allocation, no synchronisation (capturable).  The single-layer entry points run the same kernels; dbw_lpips_conv3x3 takes
 * a K-major weight wt[co][(ky*3+kx)*C_in + ci] already TF32-rounded, and optional bias, and mask (out *= [mask > 0]).
 *
 * The workspace, in floats, with H_k = H >> k, W_k = W >> k the sizes after k pools and every region starting at a
 * multiple of 64 floats (its length rounded up to a multiple of 64), in this order:
 *  - act[l], l = 0..12: rec's activation after layer l's ReLU, NHWC (B, H_k, W_k, C_out[l]) at the layer's level k
 *    (0,0, 1,1, 2,2,2, 3,3,3, 4,4,4).  Without save_for_backward only the taps l = 1, 3, 6, 9, 12 have a region;
 *  - tap0[k], k = 0..4: imgs' taps relu1_2 .. relu5_3, NHWC (B, H_k, W_k, C_k), C_k = 64, 128, 256, 512, 512;
 *  - s0, s1: scratch of B*H*W*64 floats each;
 *  - the head partials: per tap k in order (not padded between taps), B x ceil(H_k W_k / 64) floats, partial[b][c] the sum
 *    of the head over pixels 64c .. 64c + 63 of image b (row-major), as dbw_lpips_head_forward writes it;
 *  - 64 floats whose first holds the uint32 seed the forward used (dbw_lpips_forward_cached keeps its int32 miss count in
 *    the second).
 * value[b] is sum_k (sum_c partial[b][c], in c order) * (1 / (H_k W_k) in fp32), summed over k in order.
 *
 * dbw_lpips_head_forward and dbw_lpips_head_backward run one head, as the whole term does, on NHWC features f0 (imgs) and
 * f1 (rec) of shape (B, H, W, C), C = 64, 128, 256 or 512, with lin (C) and the dropout of tap `tap` (0..4) for the seed
 * *seed when `train` (without `train`, seed may be NULL).  The forward writes partials (B, ceil(H*W / 64)) as above.  The
 * backward writes g (B, H, W, C) = (d sum_b grad_value[b] head_b / d f1 + (accumulate ? g : 0)) * [f1 > 0], head_b being the
 * spatial mean of image b's head.
 */
typedef struct DbwLpipsNet {
  const float* conv_w[13];
  const float* conv_b[13];
  const float* lin_w[5];
  const float* shift;
  const float* scale;
  void* prepared;
} DbwLpipsNet;

int dbw_lpips_workspace_bytes(int64_t B, int32_t H, int32_t W, int32_t save_for_backward, size_t* workspace_bytes,
                              size_t* prepared_bytes);
int dbw_lpips_prepare_weights(const DbwLpipsNet* net, void* stream);
int dbw_lpips_forward(const DbwLpipsNet* net, const float* in0, const float* in1, int64_t B, int32_t H, int32_t W, int32_t normalize,
                      int32_t train, int32_t save_for_backward, uint32_t* seed, float* value, void* workspace,
                      size_t workspace_bytes, void* stream);
int dbw_lpips_backward(const DbwLpipsNet* net, const float* grad_value, int64_t B, int32_t H, int32_t W, int32_t normalize,
                       int32_t train, float* grad_in1, void* workspace, size_t workspace_bytes, void* stream);
int dbw_lpips_conv3x3(const float* in, const float* wt, const float* bias, const float* mask, float* out, int64_t B, int32_t H,
                      int32_t W, int32_t C_in, int32_t C_out, int32_t relu, void* stream);
int dbw_lpips_conv_first(const float* x, const float* w, const float* bias, const float* shift, const float* scale, int32_t normalize,
                         float* out, int64_t B, int32_t H, int32_t W, void* stream);
int dbw_lpips_dgrad_last(const float* g, const float* w, const float* scale, int32_t normalize, float* out, int64_t B, int32_t H,
                         int32_t W, void* stream);
int dbw_lpips_maxpool(const float* in, float* out, int64_t B, int32_t H, int32_t W, int32_t C, void* stream);
int dbw_lpips_maxpool_backward(const float* in, const float* gout, float* gin, int64_t B, int32_t H, int32_t W, int32_t C,
                               void* stream);
int dbw_lpips_head_forward(const float* f0, const float* f1, const float* lin, int64_t B, int32_t H, int32_t W, int32_t C,
                           int32_t tap, int32_t train, const uint32_t* seed, float* partials, void* stream);
int dbw_lpips_head_backward(const float* f0, const float* f1, const float* lin, int64_t B, int32_t H, int32_t W, int32_t C,
                            int32_t tap, int32_t train, const uint32_t* seed, const float* grad_value, int32_t accumulate,
                            float* g, void* stream);

/*
 * LPIPS target cache: the taps of fixed in0 images (a scene's training views) computed once and read by every later call,
 * with the same results bit for bit.  The caller owns the arena, dbw_lpips_cache_bytes(H, W) per image times N bytes,
 * device memory with 256-byte alignment, laid out in floats as:
 *  - tap[k], k = 0..4: the taps relu1_2 .. relu5_3 of the N images, NHWC (N, H_k, W_k, C_k), as tap0[k] of the workspace;
 *  - N uint64 fingerprints (csrc/dbw_lpips_cache.cuh);
 *  - a copy of the N images (N, 3, H, W).
 * The taps are those of the per-call forward to the bit: every convolution row depends only on its own image and the
 * weights, its tile shape only on C_out and its K order only on C_in, whatever the batch and the image's place in it.
 *
 * dbw_lpips_cache_targets fills the arena of `cache` from imgs (N, 3, H, W) for cache->normalize, `chunk` images at a time,
 * in a workspace of dbw_lpips_workspace_bytes(chunk, H, W, 0) bytes.  It uses the prepared weights: register again (or
 * drop the cache) whenever the weights change.
 *
 * dbw_lpips_forward_cached is dbw_lpips_forward with in0 looked up in the cache: each image's fingerprint selects the
 * entries with the same fingerprint, and the first whose stored image is equal bit for bit is a hit.  It writes route
 * (B, 2) int32: route[b][0] = the entry of a hit, or -(s + 1) for miss slot s (misses numbered in b order); route[s][1] =
 * the image of miss slot s (-1 past the misses).  The conv chain of in0 runs over the misses only (every kernel bounded by
 * the device miss count, kept in the second float of the workspace's seed region), their taps in the first slots of tap0;
 * the heads read f0 per route, the dropout keyed on b as always.  n_hits (optional, one int32) receives the hit count.
 * dbw_lpips_backward_cached is dbw_lpips_backward with the route and cache of that forward.  Both need the cache's H, W and
 * normalize equal to the call's, run on `stream` only and are capturable: a captured call looks its inputs up on every
 * replay.  The workspace is that of dbw_lpips_workspace_bytes.
 */
typedef struct DbwLpipsTargetCache {
  void* arena;
  int64_t N;
  int32_t H, W;
  int32_t normalize;
} DbwLpipsTargetCache;

int dbw_lpips_cache_bytes(int32_t H, int32_t W, size_t* bytes_per_image);
int dbw_lpips_cache_targets(const DbwLpipsNet* net, const float* imgs, const DbwLpipsTargetCache* cache, int64_t chunk, void* workspace,
                            size_t workspace_bytes, void* stream);
int dbw_lpips_forward_cached(const DbwLpipsNet* net, const DbwLpipsTargetCache* cache, const float* in0, const float* in1, int64_t B,
                             int32_t H, int32_t W, int32_t normalize, int32_t train, int32_t save_for_backward, uint32_t* seed,
                             float* value, int32_t* route, int32_t* n_hits, void* workspace, size_t workspace_bytes, void* stream);
int dbw_lpips_backward_cached(const DbwLpipsNet* net, const DbwLpipsTargetCache* cache, const int32_t* route, const float* grad_value,
                              int64_t B, int32_t H, int32_t W, int32_t normalize, int32_t train, float* grad_in1, void* workspace,
                              size_t workspace_bytes, void* stream);

/*
 * VGG16 feature-reconstruction loss: the reference's PerceptualLoss (src/model/loss.py:66-111, `perceptual_name:
 * perceptual`), on the LPIPS kernels above.  in0 (imgs), in1 (rec): (B,3,H,W) fp32 NCHW, 1 <= B <= 65535,
 * B*H*W < 2^31 - 128, 2^(L-1) <= H, W <= 32767 for the deepest requested level L (its tap is then at least 1x1).
 *   levels              bit k-1 set: level k used, k = 1..5 (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3); 1..31.
 *   normalize_input     the first layer reads (x - shift) / scale, shift = mean_rgb, scale = std_rgb (net->shift, ->scale);
 *                       0: x as is (shift and scale may then be NULL).  LPIPS's 2x - 1 is never applied.
 *   normalize_features  f / (||f||_2 over channels + 1e-10) before the difference (the LPIPS head with weight w and no
 *                       dropout; an all-zero feature vector gets no normalisation gradient); 0: f as is.
 *   sum_channels        w = 1: the squared difference summed over channels, averaged over pixels; 0: w = 1 / C_k, the
 *                       average over C_k*H_k*W_k.
 * value[b] = sum over the requested levels k, in increasing order, of (sum_c partial[b][c], in c order) * (1 / (H_k W_k)
 * in fp32), partial[b][c] the sum of w * (f0 - f1)^2 over channels and pixels 64c .. 64c + 63 of image b's level k.  The
 * trunk runs only through the deepest requested level (level 3: convolutions 0..6 and two pools), in the arithmetic of the
 * LPIPS trunk.  conv_w, conv_b and `prepared` of `net` as for LPIPS (dbw_lpips_prepare_weights; lin_w is not read and may
 * be NULL).
 *
 * dbw_vgg_loss_forward writes value (B); with save_for_backward it keeps what dbw_vgg_loss_backward needs.
 * dbw_vgg_loss_backward writes grad_in1 (B,3,H,W) = sum_b grad_value[b] d value[b] / d in1 from the workspace of a
 * save_for_backward forward with the same options (the workspace untouched in between).  Both run on `stream` only: no
 * allocation, no synchronisation (capturable).
 *
 * The workspace (dbw_vgg_loss_workspace_bytes for the same B, H, W, options and save_for_backward), in floats, every region
 * starting at a multiple of 64 floats (its length rounded up to a multiple of 64), in this order:
 *  - act[l], l = 0..last (last = 1, 3, 6, 9, 12 for L = 1..5): rec's activation after layer l's ReLU, NHWC, as for LPIPS.
 *    Without save_for_backward only the taps of the requested levels have a region;
 *  - tap0[k] for the requested levels k, in order: imgs' tap, NHWC (B, H_k, W_k, C_k);
 *  - s0, s1: scratch of B*H*W*64 floats each;
 *  - the head partials: per requested level in order (not padded between levels), B x ceil(H_k W_k / 64) floats;
 *  - 2568 constants the forward writes: per level k, 512 floats whose first C_k hold w; then shift 0 and scale 1 (4 floats
 *    each), the identity transform used without normalize_input.
 */
typedef struct DbwVggLossOptions {
  int32_t levels;
  int32_t normalize_input;
  int32_t normalize_features;
  int32_t sum_channels;
} DbwVggLossOptions;

int dbw_vgg_loss_workspace_bytes(int64_t B, int32_t H, int32_t W, const DbwVggLossOptions* opt, int32_t save_for_backward,
                                 size_t* workspace_bytes);
int dbw_vgg_loss_forward(const DbwLpipsNet* net, const DbwVggLossOptions* opt, const float* in0, const float* in1, int64_t B,
                         int32_t H, int32_t W, int32_t save_for_backward, float* value, void* workspace, size_t workspace_bytes,
                         void* stream);
int dbw_vgg_loss_backward(const DbwLpipsNet* net, const DbwVggLossOptions* opt, const float* grad_value, int64_t B, int32_t H,
                          int32_t W, float* grad_in1, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DBW_RENDER_H */
