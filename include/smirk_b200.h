/*
 * smirk_b200 — C ABI of the H100-native SMIRK hot path (encode -> FLAME -> render -> generator).
 *
 * The reference (georgeretsi/smirk) is pure Python and has no FFI of its own; its only native seams
 * on this path are third-party: `timm.create_model` (src/smirk_encoder.py:7-12), ATen/cuDNN ops, and
 * `pytorch3d.renderer.mesh.rasterize_meshes` (src/renderer/renderer.py:185-193).  Each entry point
 * below replaces the body of one reference nn.Module.forward; the Python classes in smirk_b200/ keep
 * the reference signatures and call these through ctypes (see INTEGRATION.md for the binding).
 *
 * Conventions
 *   - return 0 = OK, <0 = argument/shape error, >0 = cudaError_t; message via smk_last_error()
 *     (thread-local).  No exceptions, no exit().
 *   - `*_create` take HOST pointers to fp32 / int32 constant arrays, fold/pack them and upload to the
 *     CURRENT CUDA device; handles are immutable afterwards.  `*_forward` take DEVICE pointers
 *     (contiguous, 16-byte aligned), never allocate, never synchronise, and order all work after / before
 *     the caller's stream (cudaStream_t passed as void*) — CUDA-graph capturable.  smk_encoder_forward
 *     runs its backbones as parallel branches that fork from and join back into that stream, using
 *     per-call fork/join events and side streams taken round-robin from a pool of 8 inside the handle:
 *     forwards are re-entrant (up to 8 in flight per encoder handle) given distinct workspaces.
 *   - the caller owns inputs, outputs and the workspace (size from `*_workspace_bytes`).
 */
#ifndef SMIRK_B200_H
#define SMIRK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SMK_VERSION 100

int smk_version(void);
const char* smk_last_error(void);

/* Launch accounting and the built-in event profiler (used by bench.py for `gpu_launches` and the
 * per-kernel roofline): smk_launch_count() = kernels launched by this library so far in the process;
 * with the profiler enabled every launch is bracketed by CUDA events on its own stream (do not enable
 * during CUDA-graph capture).  smk_profiler_report writes "tag launches total_ms bytes flops" lines
 * (algorithmic bytes / FLOPs summed over launches), returns the number of lines or -1 if buf is small. */
unsigned long long smk_launch_count(void);
void smk_profiler_enable(int on);
void smk_profiler_reset(void);
int smk_profiler_report(char* buf, size_t n);

/* ------------------------------------------------------------------------------------------------
 * FLAME  — replaces FLAME.forward (src/FLAME/FLAME.py:232-315) and lbs() (src/FLAME/lbs.py:140-227).
 * ---------------------------------------------------------------------------------------------- */
typedef struct SmkFlame SmkFlame;

typedef struct {
    int n_verts;            /* 5023 */
    int n_faces;            /* 9976 */
    int n_betas;            /* n_shape + n_exp = 350 */
    int n_joints;           /* 5, kinematic parents fixed to [-1,0,1,1,1] (FLAME.py:76-77) */
    const float* v_template;        /* [V,3]                FLAME.py:64 */
    const float* shapedirs;         /* [V,3,n_betas]        FLAME.py:67-69 */
    const float* posedirs;          /* [(J-1)*9, V*3]       FLAME.py:71-73 */
    const float* J_regressor;       /* [J,V]                FLAME.py:75 */
    const float* lbs_weights;       /* [V,J]                FLAME.py:78 */
    const float* l_eyelid;          /* [V,3]                FLAME.py:81 */
    const float* r_eyelid;          /* [V,3]                FLAME.py:82 */
    const int32_t* faces;           /* [F,3]                FLAME.py:61 */
    /* landmark embeddings (FLAME.py:94-113) */
    int n_static;  const int32_t* static_faces;  const float* static_bary;     /* 51 */
    int n_dyn_rows; int n_dyn; const int32_t* dyn_faces; const float* dyn_bary; /* 79 x 17 */
    int n_full;    const int32_t* full_faces;    const float* full_bary;       /* 68 */
    int n_mp;      const int32_t* mp_faces;      const float* mp_bary;         /* 105 */
} SmkFlameDesc;

int smk_flame_create(const SmkFlameDesc* desc, SmkFlame** out);
void smk_flame_destroy(SmkFlame* h);
size_t smk_flame_workspace_bytes(const SmkFlame* h, int B);
/* betas [B,n_betas] = cat(shape, expression); full_pose [B,15] = cat(global, neck, jaw, eyes(6));
 * eyelid [B,2] or NULL.  Outputs: verts [B,V,3]; lmk_fan [B,68,3] (17 dynamic-contour + 51 static);
 * lmk_fan3d [B,68,3]; lmk_mp [B,105,3]; joints [B,J,3] (posed joints, may be NULL);
 * dyn_idx int32 [B] (selected contour LUT row, may be NULL).                                     */
int smk_flame_forward(const SmkFlame* h, const float* betas, const float* full_pose, const float* eyelid,
                      int B, float* verts, float* lmk_fan, float* lmk_fan3d, float* lmk_mp,
                      float* joints, int32_t* dyn_idx, void* ws, size_t ws_bytes, void* stream);
/* Backward of smk_flame_forward: the gradient torch autograd takes through FLAME.forward for betas,
 * full_pose and eyelid.  dyn_idx is the forward's contour row (required).  Upstream gradients g_verts
 * [B,V,3], g_lmk_fan [B,68,3], g_lmk_fan3d [B,68,3], g_lmk_mp [B,105,3]: each may be NULL (= zero).
 * Outputs are written, not accumulated: g_betas [B,n_betas], g_full_pose [B,15], g_eyelid [B,2] (may be
 * NULL).  eyelid may be NULL.  Deterministic (no atomics).  Needs n_betas <= 350.                    */
size_t smk_flame_backward_workspace_bytes(const SmkFlame* h, int B);
int smk_flame_backward(const SmkFlame* h, const float* betas, const float* full_pose, const float* eyelid,
                       int B, const int32_t* dyn_idx,
                       const float* g_verts, const float* g_lmk_fan, const float* g_lmk_fan3d, const float* g_lmk_mp,
                       float* g_betas, float* g_full_pose, float* g_eyelid, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Renderer — replaces Renderer.forward/render/rasterize (src/renderer/renderer.py:100-207,239-250),
 * util.vertex_normals/face_vertices/batch_orth_proj (src/renderer/util.py) and the third-party
 * pytorch3d rasterize_meshes call (renderer.py:185-193; blur 0, K=1, no perspective correction).
 * ---------------------------------------------------------------------------------------------- */
typedef struct SmkRenderer SmkRenderer;

typedef struct {
    int n_verts;               /* vertices of the incoming mesh (5023) */
    int n_mask;                /* rendered subset (1787 for the FLAME `face` mask; = n_verts for full head) */
    const int32_t* mask_ids;   /* [n_mask] vertex ids, order defines the sub-mesh numbering (renderer.py:71) */
    int n_faces;               /* 3408; must be < 65536 and a multiple of 4 (packed tile ranges are read 4 at a time) */
    const int32_t* faces;      /* [n_faces,3] indices into the sub-mesh (renderer.py:74) */
    int image_size;            /* 224 */
    float z_offset;            /* added to the z of the returned tverts, 0 or 10: 0 for the face mask; 10 for the full head,
                                  where the reference's in-place `z + 10` (renderer.py:140-144) lands in transformed_vertices.
                                  The rasteriser's depth is z + 10 either way. */
} SmkRendererDesc;

int smk_renderer_create(const SmkRendererDesc* desc, SmkRenderer** out);
void smk_renderer_destroy(SmkRenderer* h);
size_t smk_renderer_workspace_bytes(const SmkRenderer* h, int B);
/* verts [B,n_verts,3], cam [B,3] = (scale, tx, ty).  Outputs: rendered [B,3,S,S]; tverts [B,n_verts,3];
 * optional (NULL to skip): pix_to_face int64 [B,S,S] (packed b*n_faces+f, -1 = background),
 * bary [B,S,S,3], zbuf [B,S,S] (both -1 on background), normals [B,n_mask,3].                       */
int smk_renderer_forward(const SmkRenderer* h, const float* verts, const float* cam, int B,
                         float* rendered, float* tverts, int64_t* pix_to_face, float* bary, float* zbuf,
                         float* normals, void* ws, size_t ws_bytes, void* stream);
/* Orthographic projection of landmark sets (renderer.py:104-108): pts [B,L,3] -> out [B,L,2]. */
int smk_project_points(const float* pts, const float* cam, int B, int L, float* out_xy, void* stream);
/* Backward of smk_renderer_forward for verts and cam, from the forward's pix_to_face, bary and normals.
 * The rasteriser part is pytorch3d's rasterize_meshes backward (blur 0, K = 1, no perspective
 * correction, no zbuf / dists gradient).  g_rendered [B,3,S,S] and g_tverts [B,n_verts,3] may be NULL
 * (= zero).  Outputs are written: g_verts [B,n_verts,3], g_cam [B,3].  Deterministic (no atomics).   */
size_t smk_renderer_backward_workspace_bytes(const SmkRenderer* h, int B);
int smk_renderer_backward(const SmkRenderer* h, const float* verts, const float* cam, int B,
                          const int64_t* pix_to_face, const float* bary, const float* normals,
                          const float* g_rendered, const float* g_tverts, float* g_verts, float* g_cam,
                          void* ws, size_t ws_bytes, void* stream);
/* Backward of smk_project_points: g_xy [B,L,2] -> g_pts [B,L,3], g_cam [B,3] (written). */
int smk_project_points_backward(const float* pts, const float* cam, int B, int L, const float* g_xy,
                                float* g_pts, float* g_cam, void* stream);

/* ------------------------------------------------------------------------------------------------
 * SmirkEncoder — replaces SmirkEncoder.forward (src/smirk_encoder.py:123-133): three timm
 * tf_mobilenetv3_{small,large,large}_minimal_100 backbones (features_only, last feature) -> global
 * average pool -> Linear heads -> split/clamps (:34-45,66-73,95-110).
 * ---------------------------------------------------------------------------------------------- */
typedef struct SmkEncoder SmkEncoder;

typedef struct {
    /* Per backbone (0 = pose/small, 1 = shape/large, 2 = expression/large): the fp32 tensors of its
     * `encoder.*` state_dict in state_dict order with `num_batches_tracked` entries removed, i.e.
     * conv weight [Cout,Cin/groups,k,k] followed by BN weight, bias, running_mean, running_var.       */
    const float* const* tensors[3];
    int n_tensors[3];
    const float* head_w[3];    /* [6,576], [n_shape,960], [n_exp+5,960] */
    const float* head_b[3];
    int n_shape;               /* 300 */
    int n_exp;                 /* 50 */
    int precision;             /* 0 = fp32 CUDA-core GEMMs, 1 = TF32 wgmma GEMMs for the 1x1 convs,
                                  2 = 1 + inverted-residual blocks run expand-1x1 + depthwise-3x3 as one fused kernel,
                                  3 = 2 with error-compensated "3xTF32" tensor-core arithmetic (operands split into TF32
                                      head + tail, three products per term): fp32-equivalent results, the parity path */
} SmkEncoderDesc;

int smk_encoder_create(const SmkEncoderDesc* desc, SmkEncoder** out);
void smk_encoder_destroy(SmkEncoder* h);
size_t smk_encoder_workspace_bytes(const SmkEncoder* h, int B);
/* img [B,3,224,224] NCHW in [0,1].  Outputs: pose_cam [B,6], shape [B,n_shape], expr [B,n_exp+5]
 * with the clamps of smirk_encoder.py:105-108 already applied to columns n_exp..n_exp+4.           */
int smk_encoder_forward(const SmkEncoder* h, const float* img, int B, float* pose_cam, float* shape,
                        float* expr, void* ws, size_t ws_bytes, void* stream);
/* Input gradient (frozen weights, eval-mode BN).  An empty batch (B = 0) is a no-op; the backward is deterministic: no
 * atomics, fixed summation order.
 * Grad-mode forward: the same launches and bitwise the same outputs as smk_encoder_forward at every precision, plus what
 * the backward needs (the output of every ReLU, fp32 NHWC, and the pre-clamp head outputs) written into `saved`
 * (caller-owned, >= smk_encoder_saved_bytes; one buffer per forward whose gradient will be taken).
 * ws / ws_bytes: the forward workspace (smk_encoder_workspace_bytes). */
size_t smk_encoder_saved_bytes(const SmkEncoder* h, int B);
int smk_encoder_forward_saved(const SmkEncoder* h, const float* img, int B, float* pose_cam, float* shape, float* expr,
                              float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name (the reference's module path of the ReLU's BatchNorm, e.g.
 * "shape_encoder.encoder.bn1" for the stem, "shape_encoder.encoder.blocks.2.1.bn1" / ".bn2" for an inverted-residual
 * block's expand / depthwise output, or the head, "expression_encoder.expression_layers.0", for its pre-clamp output),
 * float offset, and dims [4] = B,H,W,C of the NHWC tensor (a head is 1 x 1 x n_out).  Forward order within each backbone,
 * backbones in slot order (pose, shape, expression).  Returns non-zero past the last tensor. */
int smk_encoder_saved_tensor(const SmkEncoder* h, int B, int i, const char** name, size_t* offset, int* dims);
/* Input gradient: upstream gradients of the raw outputs (pose_cam [B,6], shape [B,n_shape], expr [B,n_exp+5]; each may
 * be NULL, meaning zero, and then its backbone launches nothing) -> g_img [B,3,224,224] NCHW (written, not accumulated;
 * zero-filled when every upstream gradient is NULL).  ws >= smk_encoder_backward_workspace_bytes. */
size_t smk_encoder_backward_workspace_bytes(const SmkEncoder* h, int B);
int smk_encoder_backward(const SmkEncoder* h, int B, const float* saved, size_t saved_bytes, const float* g_pose_cam,
                         const float* g_shape, const float* g_expr, float* g_img, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * SmirkGenerator — replaces SmirkGenerator.forward (src/smirk_generator.py:51-86), eval-mode BN.
 * ---------------------------------------------------------------------------------------------- */
typedef struct SmkGenerator SmkGenerator;

typedef struct {
    int in_channels, out_channels, init_features, res_blocks;    /* 6, 3, 32, 5 (demo.py:63) */
    /* fp32 tensors of the module's state_dict in state_dict order, `num_batches_tracked` removed.    */
    const float* const* tensors;
    int n_tensors;
    int precision;             /* 0 = fp32 CUDA-core implicit GEMM, 1 = TF32 wgmma implicit GEMM */
} SmkGeneratorDesc;

int smk_generator_create(const SmkGeneratorDesc* desc, SmkGenerator** out);
void smk_generator_destroy(SmkGenerator* h);
size_t smk_generator_workspace_bytes(const SmkGenerator* h, int B);
/* x [B,in_channels,224,224] NCHW -> y [B,out_channels,224,224] NCHW in (0,1). */
int smk_generator_forward(const SmkGenerator* h, const float* x, int B, float* y,
                          void* ws, size_t ws_bytes, void* stream);
/* Input gradient (frozen weights, eval-mode BN).  An empty batch (B = 0) is a no-op; the backward is deterministic: no
 * atomics, fixed summation order.
 * Grad-mode forward: the same launches and bitwise the same y as smk_generator_forward, plus the activations the backward
 * needs (the post-ReLU output of every block conv and every ResNet conv1, fp32 NHWC) written into `saved`
 * (caller-owned, >= smk_generator_saved_bytes; one buffer per forward whose gradient will be taken).
 * ws / ws_bytes: the forward workspace (smk_generator_workspace_bytes). */
size_t smk_generator_saved_bytes(const SmkGenerator* h, int B);
int smk_generator_forward_saved(const SmkGenerator* h, const float* x, int B, float* y, float* saved, size_t saved_bytes,
                                void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name (the reference's layer name, e.g. "enc1conv2", "res0conv1", "dec1conv2"),
 * float offset, and dims [4] = B,H,W,C of the NHWC tensor.  Returns non-zero past the last tensor. */
int smk_generator_saved_tensor(const SmkGenerator* h, int B, int i, const char** name, size_t* offset, int* dims);
/* Input gradient: y (the forward's output) and g_y [B,out_channels,224,224] NCHW -> g_x [B,in_channels,224,224] NCHW
 * (written, not accumulated).  ws >= smk_generator_backward_workspace_bytes. */
size_t smk_generator_backward_workspace_bytes(const SmkGenerator* h, int B);
int smk_generator_backward(const SmkGenerator* h, int B, const float* y, const float* saved, size_t saved_bytes,
                           const float* g_y, float* g_x, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Crop / warp front and back end (SURVEY.md 8f #2) — replaces the CPU `skimage.transform.warp` calls of
 * demo.py:97 and demo_video.py:128,149 (+ BGR->RGB, /255, HWC->CHW of demo.py:103-105) for frames that are
 * already on the device.  Bilinear (order 1), mode 'constant', cval 0, clip to the source range, float64
 * arithmetic, truncation to uint8 — skimage's `_warp_fast` semantics.  m / minv: [B][9] row-major float64 3x3
 * maps from OUTPUT pixel (col,row,1) to INPUT (x,y,1) (affine rows only); ws >= smk_warp_workspace_bytes(B).
 *   smk_crop_warp      : frames uint8 [B,H,W,3] -> out float32 [B,3,S,S] = uint8 result / 255; swap_rb reverses the
 *                        channel order (BGR frame -> RGB tensor).  minv == NULL: no crop transform, the uint8 result
 *                        is cv2.resize(frame, (S, S)) with INTER_LINEAR bit for bit (demo_video.py:130-136 without
 *                        --crop; an exact 2x on both axes is cv2's INTER_AREA fast path); one launch, ws unused.
 *   smk_warp_u8        : src uint8 [B,Hs,Ws,3] -> dst uint8 [B,Hd,Wd,3].
 *   smk_f32chw_to_u8hwc: (x * 255.0f).astype(uint8) of a [B,3,S,S] float image -> [B,S,S,3] (demo_video.py:148).  */
size_t smk_warp_workspace_bytes(int B);
int smk_crop_warp(const uint8_t* frames, int B, int H, int W, const double* minv, int S, int swap_rb, float* out,
                  void* ws, size_t ws_bytes, void* stream);
int smk_warp_u8(const uint8_t* src, int B, int Hs, int Ws, const double* m, int Hd, int Wd, uint8_t* dst,
                void* ws, size_t ws_bytes, void* stream);
int smk_f32chw_to_u8hwc(const float* in, int B, int S, uint8_t* out, void* stream);

/* The output grid of the video demo (demo_video.py [--crop] [--render_orig] [--use_smirk_generator]).  An empty batch
 * (B = 0) is a no-op.
 * create_mask(cropped_kpt, (S, S)) of the reference (datasets/base_dataset.py:9-15) for each frame: pts [B,L,2] int32
 * points in crop pixels, or in frame pixels without --crop (1 <= L <= 1024), mask [B,1,S,S] float, 0 inside
 * cv2.convexHull(pts) filled by cv2.fillConvexPoly (lineType 8, shift 0) and 1 outside, bit for bit (points outside the
 * mask, negative ones, repeated or collinear points included); S <= 256. */
int smk_hull_mask(const int32_t* pts, int B, int L, int S, float* mask, void* stream);
/* Workspace of smk_video_compose with render_orig == 1 (the per-panel clip range); the other modes need none. */
size_t smk_video_workspace_bytes(int B, int n_panels);
/* grid [B, Hout, (n_panels + 1) * Wout, 3] uint8 BGR, one row of panels per frame: what demo_video.py:211-214 writes.
 *   render_orig == 1: (--crop --render_orig) Hout x Wout = H x W; panel 0 = frames [B,H,W,3] (BGR); panel k =
 *                     panels[k-1] [B,3,S,S] (RGB in [0,1]) converted to uint8 ((x * 255).astype(uint8)) and warped back
 *                     to the frame with m [B,9] (float64, row-major crop -> frame similarity, tform.params), skimage
 *                     warp semantics; crop unused.
 *   render_orig == 2: (--render_orig without --crop) Hout x Wout = H x W; panel 0 = frames; panel k =
 *                     (F.interpolate(panels[k-1], (H, W), mode='bilinear') * 255).astype(uint8): torch's
 *                     upsample_bilinear2d with align_corners = False, float32 without fused multiply-adds, evaluated per
 *                     output byte; crop, m and ws unused (may be NULL).
 *   render_orig == 0: Hout x Wout = S x S; panel 0 = crop [B,3,S,S] (the encoder's RGB input in [0,1]), panel k =
 *                     panels[k-1], both converted to uint8; frames and m unused (may be NULL).
 * Any other render_orig is an error.
 * panels: host array of n_panels (1 or 2) device pointers.  ws >= smk_video_workspace_bytes(B, n_panels) with
 * render_orig == 1. */
int smk_video_compose(const uint8_t* frames, int B, int H, int W, const float* crop, const float* const* panels, int n_panels,
                      int S, const double* m, int render_orig, uint8_t* grid, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Masking between Renderer and SmirkGenerator (SURVEY.md 8f #1; src/utils/masking.py, demo.py:138-167).
 * Random draws stay with the caller (torch); these entry points are the deterministic parts.
 *   face_weights: trans_verts [B,V,3], base_prob [F] -> weights [B,F]               (masking.py:146-160)
 *   points      : face_idx int64 [B,N], bary [B,N,3] -> npoints int64 [B,N,2] (x,y)  (masking.py:166-174)
 *   compose     : img [B,3,S,S], hull [B,1,S,S], npoints/rbound (first rbound[b] points are kept), optional
 *                 rendered_mask [B,1,S,S], noise_mult [B,3,S,S], random_centres [B,1,S,S] -> masked [B,3,S,S]  */
typedef struct SmkMasking SmkMasking;
typedef struct { int n_verts; int n_faces; const int32_t* faces; } SmkMaskingDesc;
int smk_masking_create(const SmkMaskingDesc* desc, SmkMasking** out);
void smk_masking_destroy(SmkMasking* h);
size_t smk_masking_workspace_bytes(const SmkMasking* h, int B, int S);
int smk_masking_face_weights(const SmkMasking* h, const float* trans_verts, const float* base_prob, int B,
                             float* weights, void* ws, size_t ws_bytes, void* stream);
int smk_masking_points(const SmkMasking* h, const float* trans_verts, const int64_t* face_idx, const float* bary,
                       int B, int N, int image_size, int64_t* npoints, void* stream);
/* extra_points [B,3,S,S] (nullable): masking()'s third argument given explicitly (masking.py:71; the trainer passes the
 * result of transfer_pixels) instead of img * point-mask(npoints, rbound).                                                 */
int smk_masking_compose(const SmkMasking* h, const float* img, const float* hull, const int64_t* npoints, const int64_t* rbound,
                        int N, const float* extra_points, const float* rendered_mask, const float* noise_mult, const float* random_centres,
                        int wr, int B, int S, float* masked, void* ws, size_t ws_bytes, void* stream);
/* transfer_pixels (masking.py:116-129): points int64 [B,N,2] (x, y); rbound int64 [B] or NULL; ws >= B*S*S*4 bytes.       */
int smk_masking_transfer_pixels(const float* img, const int64_t* points1, const int64_t* points2, const int64_t* rbound,
                                int B, int N, int S, float* out, void* ws, size_t ws_bytes, void* stream);
/* The whole step of demo.py:138-165 with the random draws made on the device (Philox4x32-10, keyed by rng_state[0] = seed
 * and rng_state[1] = call counter, which the call increments on the stream — graph replays draw fresh samples):
 *   face weights -> N = int(mask_ratio * ratio_mul * S * S) faces by inverse CDF (multinomial with replacement) -> uniform
 *   barycentrics -> pixel coordinates -> per-image budget rbound = N / ratio_mul * U(1, ratio_mul)^(+-1) -> point mask ->
 *   masking(img, hull, img * pmask, wr, rendered_mask = any(rendered != 0), extra_noise, random_mask = p_centre).
 * rendered [B,3,S,S] is the Renderer's output; hull [B,1,S,S] the landmark hull mask (1 outside the face).  Optional
 * debug outputs (NULL to skip) export the draws so the result can be checked against the reference's functions:
 * dbg_face_idx int64 [B,N], dbg_bary [B,N,3], dbg_npoints int64 [B,N,2], dbg_rbound int64 [B], dbg_noise [B,3,S,S],
 * dbg_centres [B,1,S,S].  ws >= smk_masking_forward_workspace_bytes(h, B, S, N).                                          */
size_t smk_masking_forward_workspace_bytes(const SmkMasking* h, int B, int S, int N);
int smk_masking_forward(const SmkMasking* h, const float* img, const float* hull, const float* trans_verts, const float* rendered,
                        const float* base_prob, int B, int S, int N, int wr, float ratio_mul, float p_centre, int extra_noise,
                        uint64_t* rng_state, float* masked, int64_t* dbg_face_idx, float* dbg_bary, int64_t* dbg_npoints,
                        int64_t* dbg_rbound, float* dbg_noise, float* dbg_centres, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Peer-mapped gather buffers: the all-gather of the final outputs across the GPUs of one node (SURVEY.md 8e; the
 * reference has no multi-GPU code) as copy-engine pushes over NVLink, which take no SM from the persistent compute
 * kernels.  Each rank: smk_peer_alloc a [world][shard] buffer, exchange the 64-byte handles (any host channel),
 * smk_peer_open every peer's handle, and after a batch smk_peer_push its packed shard into slot `rank` of every buffer
 * on a communication stream.  Allocation and mapping are set-up calls; a forward never allocates.
 * ---------------------------------------------------------------------------------------------- */
int smk_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64);
int smk_peer_free(void* ptr);
int smk_peer_open(const unsigned char* handle64, void** ptr);
int smk_peer_close(void* ptr);
int smk_peer_push(void* dst, const void* src, size_t bytes, void* stream);
/* The same copy to n destinations, spread over the fan's own streams (several copy engines / NVLink ports at once);
 * ordered after the work already on `stream`, which resumes only after every copy.                                        */
typedef struct SmkPeerFan SmkPeerFan;
int smk_peer_fan_create(int n_streams, SmkPeerFan** out);
void smk_peer_fan_destroy(SmkPeerFan* f);
int smk_peer_fan_push(SmkPeerFan* f, void* const* dsts, int n, const void* src, size_t bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Kernel-level test entry points (used by tests/ to check single convolution kernels against torch;
 * not part of the drop-in surface).  All pointers are device pointers.
 *   smk_debug_conv_f32: fp32 CUDA-core implicit GEMM.  w_kn is [K][N]; mode 0 = 1x1, 1 = 3x3 zero pad,
 *                       2 = 3x3 reflection pad; shuffle = 1 stores ConvTranspose2d(k2,s2) pixel-shuffled.
 *   smk_debug_conv_tc : TF32 wgmma implicit GEMM.  wt is [N][K]; mode 2 expects `in` to be a
 *                       [B,H+2,W+2,*] buffer whose halo was filled by smk_debug_reflect_halo;
 *                       store 0 plain, 1 pixel-shuffle, 2 interior of a padded [B,H+2,W+2,*] buffer.
 * ---------------------------------------------------------------------------------------------- */
int smk_debug_conv_f32(const float* in, int ld_in, int B, int H, int W, int Cin, const float* w_kn, const float* scale,
                       const float* bias, int N, int K, int mode, int relu, const float* res, int ld_res,
                       float* out, int ld_out, int shuffle, void* stream);
int smk_debug_conv_tc(const float* in, int ld_in, int B, int H, int W, int Cin, const float* wt, const float* scale,
                      const float* bias, int N, int K, int mode, int relu, const float* res, int ld_res, int res_pad,
                      float* out, int ld_out, int store, void* stream);
int smk_debug_reflect_halo(float* buf, int B, int H, int W, int C, void* stream);
/*   smk_debug_xdw: fused expand-1x1 (TF32 wgmma) + BN + ReLU + depthwise-3x3 (fp32) + BN + ReLU of a
 *                  MobileNetV3 inverted-residual block.  x [B,H,W,Cin] NHWC; w1t [mid][Cin]; wdw [9][mid];
 *                  out [B,ceil(H/stride),ceil(W/stride),mid]; TF-SAME padding.                            */
int smk_debug_xdw(const float* x, int B, int H, int W, int Cin, const float* w1t, const float* scale1, const float* bias1,
                  int mid, const float* wdw, const float* scale2, const float* bias2, int stride, int round_out,
                  float* out, void* stream);

/*   smk_debug_conv3_win: the persistent windowed TF32 wgmma 3x3 convolution of the high-resolution narrow layers
 *                  (zero padding 1, N in {32, 64}, Cin % 32 == 0, W >= 56, resident weights <= 72 KB); wt is [N][9*Cin].      */
int smk_debug_conv3_win(const float* in, int ld_in, int B, int H, int W, int Cin, const float* wt, const float* scale,
                        const float* bias, int N, int relu, float* out, int ld_out, void* stream);
/*   smk_debug_gemm_tc3x / smk_debug_xdw3x: the error-compensated 3xTF32 variants of the two tensor-core encoder kernels
 *                  (encoder precision 3).  wt_hi / wt_lo (w1t_hi / w1t_lo) are the TF32 heads and tails of the weights:
 *                  hi = tf32(w), lo = tf32(w - hi).  in is [M, ld_in] row-major; out [M, ld_out].                       */
int smk_debug_gemm_tc3x(const float* in, int ld_in, int M, const float* wt_hi, const float* wt_lo, const float* scale,
                        const float* bias, int N, int K, int relu, const float* res, int ld_res, float* out, int ld_out, void* stream);
int smk_debug_xdw3x(const float* x, int B, int H, int W, int Cin, const float* w1t_hi, const float* w1t_lo, const float* scale1,
                    const float* bias1, int mid, const float* wdw, const float* scale2, const float* bias2, int stride,
                    float* out, void* stream);

/*   smk_debug_stem_ds: fused stem conv (3x3 s2, 3 -> 16) + BN + ReLU + depthwise-separable block 0 (fp32 CUDA cores).
 *                      img [B,3,H,W] NCHW; stem_w [27][16] (k = (c*3+ky)*3+kx); dw_w [9][16]; pw_w [16 ci][16 co];
 *                      out [B,H/2/stride,W/2/stride,16] NHWC; the skip connection is added when stride == 1.          */
int smk_debug_stem_ds(const float* img, int B, int H, int W, const float* stem_w, const float* stem_s, const float* stem_b,
                      const float* dw_w, const float* dw_s, const float* dw_b, const float* pw_w, const float* pw_s,
                      const float* pw_b, int stride, int round_out, float* out, void* stream);

#ifdef __cplusplus
}
#endif

/* SmirkEncoder train mode (batch-statistics BatchNorm and parameter gradients): include/smirk_b200_train.h. */
#include "smirk_b200_train.h"

#endif /* SMIRK_B200_H */
