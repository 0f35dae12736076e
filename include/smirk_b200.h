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
/* Train mode (BatchNorm over batch statistics, the reference trainer's encoder.train(), base_trainer.py:108-111) and the
 * gradients of every parameter (src/smirk_trainer.py:34-73).
 * A train handle holds the topology only — the backbones in `backbones` (bit set: 1 pose, 2 shape, 4 expression), the head
 * widths and the precision (as SmkEncoderDesc's; precision 2 computes as 1, there is no fused train kernel) — and is
 * destroyed by smk_encoder_destroy.  Every call reads the parameters through the device pointers of SmkEncoderTrainArgs and
 * repacks the 1x1 weights into the workspace, so an optimizer step needs no new handle.  Calls never allocate or
 * synchronise, use no float atomics (bitwise reproducible) and are CUDA-graph capturable; the eval entry points above reject
 * a train handle.  BatchNorm couples the images of a batch: outputs are not independent of the other images. */
typedef struct {
    /* Per backbone, DEVICE pointers of its `encoder.*` tensors in the order of SmkEncoderDesc.tensors (per conv: weight,
     * BN weight, bias, running_mean, running_var); running_mean / running_var are updated in place.                   */
    float* const* tensors[3];
    int n_tensors[3];
    int64_t* const* num_batches_tracked[3];   /* one per BatchNorm, in the same order; each is incremented by one     */
    const float* head_w[3];
    const float* head_b[3];
    float momentum[3];         /* running-statistics factor; negative = None (cumulative average, 1 / num_batches_tracked) */
    float eps[3];
} SmkEncoderTrainArgs;
typedef struct {
    /* Gradient outputs (written, not accumulated), NULL = not wanted.  tensors[i][j] is the gradient of
     * SmkEncoderTrainArgs.tensors[i][j]; the running-statistics entries must be NULL.  tensors[i] itself may be NULL.  */
    float* const* tensors[3];
    float* head_w[3];
    float* head_b[3];
} SmkEncoderTrainGrads;
int smk_encoder_train_create(int backbones, int n_shape, int n_exp, int precision, SmkEncoder** out);
/* Workspace of both train calls.  smk_encoder_saved_bytes / smk_encoder_saved_tensor describe the train handle's saved
 * buffer: per BatchNorm the conv's pre-BN output (named after the conv, e.g. "shape_encoder.encoder.blocks.2.1.conv_pw"),
 * every ReLU output (named as in eval mode), every block output ("...blocks.2.1"), the pooled features
 * ("shape_encoder.pooled", [B,feat]) and the heads' pre-clamp outputs, followed by the batch statistics (not listed). */
size_t smk_encoder_train_workspace_bytes(const SmkEncoder* h, int B);
/* Train-mode forward: outputs as smk_encoder_forward; updates the running statistics and num_batches_tracked of every
 * BatchNorm.  saved (>= smk_encoder_saved_bytes) keeps the activations for smk_encoder_backward_train; with saved == NULL
 * they live in ws, which must then hold smk_encoder_saved_bytes more. */
int smk_encoder_forward_train(const SmkEncoder* h, const SmkEncoderTrainArgs* args, const float* img, int B, float* pose_cam,
                              float* shape, float* expr, float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Train-mode backward from the forward's saved buffer (args and img: those of the forward).  Upstream gradients may be
 * NULL: a backbone without one, or whose parameters want no gradient while g_img is NULL, launches nothing (and writes
 * none of its gradients).  g_img [B,3,224,224] (NULL: not wanted) is written. */
int smk_encoder_backward_train(const SmkEncoder* h, const SmkEncoderTrainArgs* args, const float* img, int B, const float* saved,
                               size_t saved_bytes, const float* g_pose_cam, const float* g_shape, const float* g_expr, float* g_img,
                               const SmkEncoderTrainGrads* grads, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * SmirkGenerator — replaces SmirkGenerator.forward (src/smirk_generator.py:51-86), eval-mode BN.
 * ---------------------------------------------------------------------------------------------- */
typedef struct SmkGenerator SmkGenerator;

typedef struct {
    int in_channels, out_channels, init_features, res_blocks;    /* 6, 3, 32, 5 (demo.py:63) */
    /* fp32 tensors of the module's state_dict in state_dict order, `num_batches_tracked` removed.    */
    const float* const* tensors;
    int n_tensors;
    int precision;             /* 0 = fp32 CUDA-core implicit GEMM, 1 = TF32 wgmma implicit GEMM,
                                  3 = 1 with 3xTF32 error-compensated arithmetic (fp32-equivalent forward and input
                                  gradient on the tensor cores; the same launches as 1).  2 is not a generator precision. */
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

/* Train mode (BatchNorm over batch statistics, the reference trainer's generator.train(), base_trainer.py:108-111) and the
 * gradients of every parameter (src/smirk_trainer.py:94,295).
 * A train handle holds the topology only (the configuration and precision of SmkGeneratorDesc) and is destroyed by
 * smk_generator_destroy.  Every call reads the parameters through the device pointers of SmkGeneratorTrainArgs and repacks
 * the weights into the workspace, so an optimizer step needs no new handle.  Calls never allocate or synchronise, use no
 * float atomics (bitwise reproducible) and are CUDA-graph capturable; the eval entry points above reject a train handle.
 * BatchNorm couples the images of a batch: outputs are not independent of the other images. */
typedef struct {
    /* DEVICE pointers of the module's state_dict tensors in the order of SmkGeneratorDesc.tensors (num_batches_tracked
     * removed); running_mean / running_var are updated in place.                                                      */
    float* const* tensors;
    int n_tensors;
    int64_t* const* num_batches_tracked;   /* one per BatchNorm, in state_dict order; each is incremented by one */
    float momentum;            /* running-statistics factor of every BatchNorm; negative = None (1 / num_batches_tracked) */
    float eps;
} SmkGeneratorTrainArgs;
typedef struct {
    /* Gradient outputs (written, not accumulated), NULL = not wanted: tensors[j] is the gradient of
     * SmkGeneratorTrainArgs.tensors[j]; the running-statistics entries must be NULL.                                  */
    float* const* tensors;
} SmkGeneratorTrainGrads;
int smk_generator_train_create(int in_channels, int out_channels, int init_features, int res_blocks, int precision, SmkGenerator** out);
/* Workspace of both train calls.  smk_generator_saved_bytes / smk_generator_saved_tensor describe the train handle's saved
 * buffer: the NHWC input ("input", channels zero-padded), per conv its pre-BN output (named after the conv, e.g.
 * "enc1conv1", "res0conv2") and per BatchNorm its (+ residual) (+ ReLU) output (named after the BatchNorm, e.g.
 * "enc1norm1", "res0norm2"), each decoder's input ("dec1cat": torch.cat((upconv1 output, enc1norm2 output))) and each
 * pool's output ("pool1"), followed by the batch statistics (not listed). */
size_t smk_generator_train_workspace_bytes(const SmkGenerator* h, int B);
/* Train-mode forward: x [B,in_channels,224,224] -> y as smk_generator_forward; updates the running statistics and
 * num_batches_tracked of every BatchNorm.  saved (>= smk_generator_saved_bytes) keeps the activations for
 * smk_generator_backward_train; with saved == NULL they live in ws, which must then hold smk_generator_saved_bytes more. */
int smk_generator_forward_train(const SmkGenerator* h, const SmkGeneratorTrainArgs* args, const float* x, int B, float* y,
                                float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Train-mode backward from the forward's saved buffer and output y (args: those of the forward).  g_y [B,out_channels,
 * 224,224]; g_x [B,in_channels,224,224] (NULL: not wanted, and the first conv's dgrad does not run) is written. */
int smk_generator_backward_train(const SmkGenerator* h, const SmkGeneratorTrainArgs* args, int B, const float* y, const float* saved,
                                 size_t saved_bytes, const float* g_y, float* g_x, const SmkGeneratorTrainGrads* grads, void* ws,
                                 size_t ws_bytes, void* stream);

/* Test entry point of the train path's 3x3 weight gradient (tests/test_gpu_generator_train_kernels.py; not part of the
 * drop-in surface).  Device pointers; it calls the host helper the train backward uses.  g [B,H,W,cout] (the gradient
 * of the conv's output), a [B,H,W,lda] (the conv's input, its first cin channels) -> out [cout][cin][3][3] (torch's
 * layout), 3x3 stride 1 with zero padding 1 (reflect 0) or ReflectionPad2d(1) (reflect 1).  ws: kWgradPart floats
 * (16 MiB) of split-K partials. */
int smk_debug_train_conv3_wgrad(const float* g, const float* a, int lda, int B, int H, int W, int cin, int cout, int reflect, float* out,
                                void* ws, size_t ws_bytes, void* stream);

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

/* The reference trainer's masking and the cycle path's parameter augmentation, with every random draw made on the device.
 * Randomness: a counter-based generator (Philox4x32-10) keyed by rng_state = {seed, call counter}, two uint64 in device
 * memory.  Every call advances the counter on the stream, so a captured CUDA graph draws fresh numbers on every replay
 * and a given (seed, counter) always gives the same bits.  The draws are equal in distribution to the reference's torch
 * draws, not equal to them; given the draws the optional debug pointers export, every output equals the reference's
 * fp32 arithmetic bit for bit.  Calls never allocate or synchronise with the host and are CUDA-graph capturable. */
/* ---- the trainer's masking (src/smirk_trainer.py:76-92 step1, :262-293 step2), on a SmkMasking handle ----
 * N = int(mask_ratio * S * S) points per image, all of them kept (no rbound budget); faces by inverse CDF of the face
 * weights (masking.py:146-160) of tv_first [B,V,3], uniform reflected barycentrics.  R = Ke * B output rows; row r uses
 * the draws, image, hull and tv_first points of row r mod B (torch's .repeat(Ke)).
 *   step 1 (Ke == 1, tv_second NULL): points = points(tv_first); extra = transfer_pixels(img, points, points);
 *           masked = masking(img, hull, extra, wr, rendered_mask = 1 - all(rendered == 0), extra_noise, random_mask = p_centre)
 *   step 2: points1 = points(tv_first), points2 = points(tv_second [R,V,3]);
 *           extra = transfer_pixels(img.repeat(Ke), points1.repeat(Ke), points2)   (duplicate targets: the last pair wins)
 *           masked = masking(img.repeat(Ke), hull.repeat(Ke), extra, wr, rendered_mask = all(rendered > 0), extra_noise,
 *                            random_mask = p_centre)
 * img [B,3,S,S], hull [B,1,S,S], rendered [R,3,S,S] (step 2: the second path's render), base_prob [F]; masked [R,3,S,S].
 * Debug outputs (each nullable): face_idx int64 [B,N], bary [B,N,3], points1 int64 [B,N,2] (x, y), points2 int64 [R,N,2]
 * (step 2 only), noise_mult [R,3,S,S] (randn * 0.05 + 1), centres [R,1,S,S] (Bernoulli(p_centre) patch centres). */
size_t smk_masking_train_workspace_bytes(const SmkMasking* h, int B, int Ke, int S, int N);
int smk_masking_train_forward(const SmkMasking* h, int step, const float* img, const float* hull, const float* tv_first,
                              const float* tv_second, const float* rendered, const float* base_prob, int B, int Ke, int S, int N,
                              int wr, float p_centre, uint64_t* rng_state, float* masked, int64_t* dbg_face_idx, float* dbg_bary,
                              int64_t* dbg_points1, int64_t* dbg_points2, float* dbg_noise, float* dbg_centres, void* ws,
                              size_t ws_bytes, void* stream);

/* ---- the cycle path's parameter augmentation (src/smirk_trainer.py:189-248) ----
 * Templates (src/utils/utils.py:load_templates): n_keys keys in dict order; key k owns rows row_offset[k] ..
 * row_offset[k+1]-1 of rows [total][n_exp] (fp32, each row the first n_exp values of a template cast from fp64).     */
typedef struct SmkCycle SmkCycle;
typedef struct {
    int n_keys;
    const int32_t* row_offset;   /* host [n_keys + 1], row_offset[0] = 0, strictly increasing */
    const float* rows;           /* host [row_offset[n_keys]][n_exp]                          */
    int n_exp;                   /* num_expression: the columns a template injection overwrites  */
} SmkCycleDesc;
/* Every field nullable; R = Ke * B, groups of sizes n0 = R/4, n1 = 2R/4 - R/4, n2 = 3R/4 - 2R/4, n3 = R - 3R/4 (floors),
 * E = the expression width.  Group-indexed draws are in group order (row k of group g is output row gids[start_g + k]). */
typedef struct {
    int64_t* gids;          /* [R]  the group permutation (torch.randperm(R))              */
    int64_t* perm1;         /* [n1] the in-group permutation of group 1                     */
    float* param_mask;      /* [n0,E] Bernoulli(0.5)                                        */
    float* jaw_mask;        /* [R]    Bernoulli(0.5) of the jaw's scale_mask                */
    float* randn0a;         /* [n0,E] group 0: the normal of new_expressions               */
    float* randn0b;         /* [n0,E] group 0: the normal of the extra noise               */
    float* randn1;          /* [n1,E] */
    float* randn2;          /* [n2,E] */
    float* randn3;          /* [n3,E] */
    float* randn_jaw;       /* [R,3]  */
    float* rand0a;          /* [n0]   U(0,1) draws: group 0's scale of new_expressions (1 + 2U) */
    float* rand0b;          /* [n0]   group 0's noise scale (0.2U)                          */
    float* rand1a;          /* [n1]   group 1's expression scale (0.25 + 1.25U)             */
    float* rand1b;          /* [n1]   group 1's noise scale                                 */
    float* rand2a;          /* [n2]   group 2's template scale (0.25 + 1.25U)               */
    float* rand2b;          /* [n2]   group 2's noise scale                                 */
    float* rand3;           /* [n3]   group 3's noise scale                                 */
    float* rand_eyelid;     /* [R,2]  the eyelid tweak (use_eyelids)                        */
    float* rand3_eyelid;    /* [n3,2] group 3's eyelids                                     */
    int64_t* tmpl_key;      /* [n2]   key index of each template pick                       */
    int64_t* tmpl_row;      /* [n2]   row within that key                                   */
} SmkCycleDraws;
int smk_cycle_create(const SmkCycleDesc* desc, SmkCycle** out);
void smk_cycle_destroy(SmkCycle* h);
/* Encoder outputs [B, dim] (dims[0..5]: pose, cam, shape, expression, jaw (3), eyelid (2)) -> flame_feats [Ke*B, dim]:
 * pose, cam and shape copied from row r mod B; expression, jaw and eyelid augmented as the reference does.  One launch. */
int smk_cycle_augment(const SmkCycle* h, const float* const* in, float* const* out, const int* dims, int B, int Ke, int use_eyelids,
                      uint64_t* rng_state, const SmkCycleDraws* dbg, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The trainer's frozen networks: VGGPerceptualLoss, MICA and ExpressionLoss.  create takes the host fp32 tensors of the
 * module's state_dict (which ones: at each network) and uploads them to the current device; the weights are frozen and
 * every BatchNorm runs in eval mode.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const float* const* tensors;   /* host fp32 tensors, in state_dict order */
    int n_tensors;
    int precision;             /* 0 = fp32 CUDA-core implicit GEMM, 1 = TF32 wgmma implicit GEMM,
                                  3 = 1 with 3xTF32 error-compensated arithmetic (fp32-equivalent).  2 is not a precision. */
} SmkNetDesc;

/* VGGPerceptualLoss (src/losses/VGGPerceptualLoss.py) — replaces VGGPerceptualLoss.forward: sum over the taps relu1_2,
 * relu2_2, relu3_3, relu4_3 of torchvision VGG16 features[:23] of l1_loss(phi(x), phi(y)), x and y normalised as
 * (v * 0.5 + 0.5 - mean) / std.  The input gradient goes to x, y or both.
 * Tensors (22): mean [1,3,1,1], std [1,3,1,1], then weight [cout,cin,3,3] and bias [cout] of the ten convolutions
 * (blocks.0.0 ... blocks.3.21). */
typedef struct SmkVggLoss SmkVggLoss;
int smk_vgg_loss_create(const SmkNetDesc* desc, SmkVggLoss** out);
void smk_vgg_loss_destroy(SmkVggLoss* h);
size_t smk_vgg_loss_workspace_bytes(const SmkVggLoss* h, int B);
/* x, y [B,3,224,224] NCHW -> loss, one fp32 device scalar (written).  x and y may be the same tensor.  Deterministic:
 * no atomics, fixed summation order.  An empty batch (B = 0) is an argument error: the loss of nothing is undefined. */
int smk_vgg_loss_forward(const SmkVggLoss* h, const float* x, const float* y, int B, float* loss,
                         void* ws, size_t ws_bytes, void* stream);
/* Grad-mode forward: the same launches and bitwise the same loss, plus what the backward needs in `saved` (caller-owned,
 * >= smk_vgg_loss_saved_bytes): the post-ReLU output of every convolution, fp32 NHWC, for each half whose gradient is
 * wanted, and per tap an int8 map of sign(phi(x) - phi(y)) (-1, 0, +1).  need: 1 = gradient to x, 2 = to y, 3 = both.
 * ws / ws_bytes: the forward workspace (smk_vgg_loss_workspace_bytes). */
size_t smk_vgg_loss_saved_bytes(const SmkVggLoss* h, int B, int need);
int smk_vgg_loss_forward_saved(const SmkVggLoss* h, const float* x, const float* y, int B, int need, float* loss,
                               float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name ("relu1_1" ... "relu4_3": fp32, dims B' = B per saved half (x's first when both),
 * "sign1_2" ... "sign4_3": int8, dims B), offset in floats, and dims [4] = B,H,W,C of the NHWC tensor.  Returns non-zero
 * past the last tensor. */
int smk_vgg_loss_saved_tensor(const SmkVggLoss* h, int B, int need, int i, const char** name, size_t* offset, int* dims);
/* Input gradient of the loss times the device scalar g: g_x and g_y [B,3,224,224] NCHW (written, not accumulated; the one
 * `need` does not ask for may be null).  `need` and `saved` are those of the grad-mode forward.
 * ws >= smk_vgg_loss_backward_workspace_bytes. */
size_t smk_vgg_loss_backward_workspace_bytes(const SmkVggLoss* h, int B, int need);
int smk_vgg_loss_backward(const SmkVggLoss* h, int B, int need, const float* saved, size_t saved_bytes, const float* g,
                          float* g_x, float* g_y, void* ws, size_t ws_bytes, void* stream);

/* MICA (src/models/MICA/mica.py): the frozen ArcFace iResNet-100 and shape regressor the pretraining step's MICA shape loss
 * runs, forward only, and that loss, mse_loss(shape_params, mica_shape), with its gradient to shape_params.
 * Tensors (781): the state_dict without num_batches_tracked: arcface.* (conv1, bn1, prelu, layer1.0 ... layer4.2, bn2,
 * fc, features), then regressor.* (network.0 ... network.3, output). */
typedef struct SmkMica SmkMica;
int smk_mica_create(const SmkNetDesc* desc, SmkMica** out);
void smk_mica_destroy(SmkMica* h);
size_t smk_mica_workspace_bytes(const SmkMica* h, int B);
/* images [B,3,112,112] NCHW (RGB in [0, 1]) -> shape_params [B,300]; features (optional, null: not written) [B,512]: the
 * ArcFace embedding before F.normalize.  Eval-mode BatchNorm throughout.  Deterministic and batch-independent. */
int smk_mica_forward(const SmkMica* h, const float* images, int B, float* shape_params, float* features,
                     void* ws, size_t ws_bytes, void* stream);
/* MICA shape loss over the first D columns: loss (one fp32 device scalar, written) = mean over b < B, d < D of
 * (shape_params[b*D + d] - mica_shape[b*ld + d])^2.  One CTA, fixed summation order, no atomics. */
int smk_mica_shape_loss_forward(const float* shape_params, const float* mica_shape, int B, int D, int ld, float* loss,
                                void* stream);
/* Its gradient times the device scalar g: grad [B,D] (written) = (2 / (B*D)) * (shape_params - mica_shape) * g. */
int smk_mica_shape_loss_backward(const float* shape_params, const float* mica_shape, int B, int D, int ld, const float* g,
                                 float* grad, void* stream);

/* ExpressionLoss (src/losses/ExpressionLoss.py) — replaces ExpressionLoss.forward(gen, tar, use_mean, metric):
 * f = backbone(x).view(B, -1), EMOCA's eval-mode ResNet-50 (Bottleneck layers (3, 4, 6, 3), the stride of each layer's
 * first block on its 3x3 conv) up to the 7x7 average pool, on gen and tar [B,3,224,224] as they are; per face
 * l2 = mean((f_gen - f_tar)^2), l1 = mean(|.|) or cos = 1 - cosine_similarity (eps 1e-8); use_mean: their mean over the
 * faces.  The input gradient goes to gen, tar or both.
 * Tensors (265): backbone.* in state_dict order, num_batches_tracked and backbone.fc.* left out: conv1.weight, bn1
 * (weight, bias, running_mean, running_var), then per Bottleneck conv1, conv2, bn1, bn2, conv3, bn3 and, in the first
 * block of each layer, downsample.0 and downsample.1. */
typedef struct SmkExpressionLoss SmkExpressionLoss;
int smk_expression_loss_create(const SmkNetDesc* desc, SmkExpressionLoss** out);
void smk_expression_loss_destroy(SmkExpressionLoss* h);
size_t smk_expression_loss_workspace_bytes(const SmkExpressionLoss* h, int B);
/* gen, tar [B,3,224,224] NCHW -> loss: [B] per-face values, or one scalar (their mean) when use_mean.  metric: 0 = l2,
 * 1 = l1, 2 = cos.  features (optional): [2B,2048], gen's then tar's.  Deterministic: no atomics, fixed summation
 * orders; face b's value does not depend on the other faces. */
int smk_expression_loss_forward(const SmkExpressionLoss* h, const float* gen, const float* tar, int B, int metric, int use_mean,
                                float* loss, float* features, void* ws, size_t ws_bytes, void* stream);
/* Grad-mode forward: the same launches and bitwise the same loss, plus what the backward needs in `saved` (caller-owned,
 * >= smk_expression_loss_saved_bytes): for each image whose gradient is wanted, the pool output and its int8 argmax tap,
 * and u1, u2 (the post-ReLU outputs of conv1 and conv2) and y of every block, fp32 NHWC; then both halves' features.
 * need: 1 = gradient to gen, 2 = to tar, 3 = both.  ws / ws_bytes: the forward workspace. */
size_t smk_expression_loss_saved_bytes(const SmkExpressionLoss* h, int B, int need);
int smk_expression_loss_forward_saved(const SmkExpressionLoss* h, const float* gen, const float* tar, int B, int metric, int use_mean,
                                      int need, float* loss, float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name ("pool", "pool_argmax" (int8), "layer1.0.u1" ... "layer4.2.y", dims B' = B per
 * saved half, gen's first when both; last "features", dims [2B,1,1,2048]), offset in floats, and dims [4] = B,H,W,C of
 * the NHWC tensor.  Returns non-zero past the last tensor. */
int smk_expression_loss_saved_tensor(const SmkExpressionLoss* h, int B, int need, int i, const char** name, size_t* offset, int* dims);
/* Input gradient of the loss times g ([B], or one scalar when use_mean): g_gen and g_tar [B,3,224,224] NCHW (written,
 * not accumulated; the one `need` does not ask for may be null).  metric, use_mean, need and saved are those of the
 * grad-mode forward.  ws >= smk_expression_loss_backward_workspace_bytes. */
size_t smk_expression_loss_backward_workspace_bytes(const SmkExpressionLoss* h, int B, int need);
int smk_expression_loss_backward(const SmkExpressionLoss* h, int B, int metric, int use_mean, int need, const float* saved,
                                 size_t saved_bytes, const float* g, float* g_gen, float* g_tar, void* ws, size_t ws_bytes,
                                 void* stream);

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

/* ------------------------------------------------------------------------------------------------
 * Train-kernel test entry points (used by tests/ to check the train-mode kernels one at a time against torch; not
 * part of the drop-in surface).  All pointers are device pointers; each calls the host helper the train calls use, so
 * the launches are theirs.  Activations are NHWC [M = B*H*W, C]; weights are in torch's layout.  ws / ws_bytes: scratch
 * for the partial sums, at least 512 * C * 16 bytes for bn_forward, that + 8 * C for bn_backward, and 16 MiB (4M
 * floats) for the weight gradients.
 *   bn_forward   : batch statistics of z -> mean, invstd; running_mean / running_var / num_batches_tracked updated as
 *                  the train forward does (momentum < 0: None); y = gamma * (z - mean) * invstd + beta (+ res) (ReLU when
 *                  relu) (TF32-rounded when round).  C % 4 == 0.
 *   bn_backward  : g (gradient of y; masked by [y > 0] when y is given) -> gz, which may alias g; g_gamma / g_beta
 *                  (either may be NULL).
 *   pw_wgrad     : out [Co][Ci] = sum over the M pixels of g[p][co] * a[p][ci].
 *   dw_*         : the 3x3 depthwise conv (TF-SAME, stride 1 or 2) of a [B,H,H,C] with w [C][1][3][3]; dgrad adds res
 *                  (may be NULL) to the input gradient [B,H,H,C].
 *   stem_*       : the stem conv of img [B,3,H,W] (3x3 stride 2 TF-SAME, 3 -> 16; H and W of one parity), z and its
 *                  gradient g [B,ceil(H/2),ceil(W/2),16]; out [16][3][3][3].
 *   head_backward: codes [n_out] (NULL: all 0) per output: 0 pass, 1 clamp [0, 1], 2 ReLU, 3 clamp [-0.2, 0.2], judged
 *                  on the pre-clamp output raw [B][n_out]; gp [B][n_out] (gradient of raw), g_feat [B,HW,C] (of the
 *                  features before the global pool), g_w [n_out][C] and g_b [n_out] (either may be NULL) from pooled [B][C].
 * ---------------------------------------------------------------------------------------------- */
int smk_debug_train_bn_forward(const float* z, int M, int C, float eps, float momentum, const float* gamma, const float* beta,
                               float* rmean, float* rvar, int64_t* nbt, const float* res, int relu, int round, float* mean,
                               float* invstd, float* y, void* ws, size_t ws_bytes, void* stream);
int smk_debug_train_bn_backward(const float* g, const float* y, const float* z, const float* mean, const float* invstd,
                                const float* gamma, int M, int C, int round, float* gz, float* g_gamma, float* g_beta, void* ws,
                                size_t ws_bytes, void* stream);
int smk_debug_train_pw_wgrad(const float* g, const float* a, int M, int Co, int Ci, float* out, void* ws, size_t ws_bytes, void* stream);
int smk_debug_train_dw_forward(const float* a, const float* w, int B, int H, int C, int stride, float* z, void* stream);
int smk_debug_train_dw_wgrad(const float* g, const float* a, int B, int H, int C, int stride, float* out, void* ws, size_t ws_bytes,
                             void* stream);
int smk_debug_train_dw_dgrad(const float* g, const float* w, const float* res, int B, int H, int C, int stride, float* out, void* stream);
int smk_debug_train_stem_forward(const float* img, const float* w, int B, int H, int W, float* z, void* stream);
int smk_debug_train_stem_wgrad(const float* g, const float* img, int B, int H, int W, float* out, void* ws, size_t ws_bytes, void* stream);
int smk_debug_train_head_backward(const float* g, const float* raw, const uint8_t* codes, const float* w, const float* pooled, int B,
                                  int n_out, int HW, int C, float* gp, float* g_feat, float* g_w, float* g_b, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SMIRK_B200_H */
