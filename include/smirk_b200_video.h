/*
 * smirk_b200 — the output grid of the video demo (demo_video.py --crop [--render_orig] [--use_smirk_generator]).
 *
 * Included at the end of smirk_b200.h, after smirk_b200_encoder_grad.h: C and C++ callers see one ABI (SMK_VERSION 100).
 * Conventions as there: status codes, caller-owned device buffers, no allocation and no synchronisation (CUDA-graph
 * capturable), an empty batch (B = 0) is a no-op.
 */
#ifndef SMIRK_B200_VIDEO_H
#define SMIRK_B200_VIDEO_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* create_mask(cropped_kpt, (S, S)) of the reference (datasets/base_dataset.py:9-15) for each frame: pts [B,L,2] int32
 * points in crop pixels (1 <= L <= 1024), mask [B,1,S,S] float, 0 inside cv2.convexHull(pts) filled by
 * cv2.fillConvexPoly (lineType 8, shift 0) and 1 outside, bit for bit (points outside the crop, repeated or collinear
 * points included); S <= 256. */
int smk_hull_mask(const int32_t* pts, int B, int L, int S, float* mask, void* stream);
/* Workspace of smk_video_compose with render_orig (the per-panel clip range); without render_orig none is needed. */
size_t smk_video_workspace_bytes(int B, int n_panels);
/* grid [B, Hout, (n_panels + 1) * Wout, 3] uint8 BGR, one row of panels per frame: what demo_video.py:211-214 writes.
 *   render_orig != 0: Hout x Wout = H x W; panel 0 = frames [B,H,W,3] (BGR); panel k = panels[k-1] [B,3,S,S] (RGB in
 *                     [0,1]) converted to uint8 ((x * 255).astype(uint8)) and warped back to the frame with m [B,9]
 *                     (float64, row-major crop -> frame similarity, tform.params), skimage warp semantics; crop unused.
 *   render_orig == 0: Hout x Wout = S x S; panel 0 = crop [B,3,S,S] (the encoder's RGB input in [0,1]), panel k =
 *                     panels[k-1], both converted to uint8; frames and m unused (may be NULL).
 * panels: host array of n_panels (1 or 2) device pointers.  ws >= smk_video_workspace_bytes(B, n_panels) with render_orig. */
int smk_video_compose(const uint8_t* frames, int B, int H, int W, const float* crop, const float* const* panels, int n_panels,
                      int S, const double* m, int render_orig, uint8_t* grid, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SMIRK_B200_VIDEO_H */
