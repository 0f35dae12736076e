/* smirk_b200 C ABI: the reference trainer's masking and the cycle path's parameter augmentation, with every random draw
 * made on the device.  Kept in a header of its own, next to include/smirk_b200.h (whose masking handle it uses), so that
 * each header's prototype list stays fixed.
 *
 * Randomness: a counter-based generator (Philox4x32-10) keyed by rng_state = {seed, call counter}, two uint64 in device
 * memory.  Every call advances the counter on the stream, so a captured CUDA graph draws fresh numbers on every replay
 * and a given (seed, counter) always gives the same bits.  The draws are equal in distribution to the reference's torch
 * draws, not equal to them; given the draws the optional debug pointers export, every output equals the reference's
 * fp32 arithmetic bit for bit.  Calls never allocate or synchronise with the host and are CUDA-graph capturable. */
#pragma once
#include "smirk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

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

#ifdef __cplusplus
}
#endif
