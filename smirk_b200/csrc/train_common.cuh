// Building blocks shared by the train-mode paths of the encoder (encoder_train.cu) and the generator (generator_train.cu):
// train-mode BatchNorm (batch statistics, running-statistics update, backward), the split-K weight-gradient reductions, and
// the per-call weight packing.  Every reduction sums over fixed pixel chunks in fixed order (fp64 where noted), with no
// atomics: results are bitwise reproducible and every launch is CUDA-graph capturable.
#pragma once
#include "conv.cuh"

namespace trn {

constexpr int kMaxChunks = 512;            // BN reductions: at most this many pixel chunks per layer
constexpr size_t kWgradPart = 1u << 22;    // floats of split-K partials of one weight gradient (see wgrad_chunks)

// One BatchNorm's device tensors: the conv weight before it, its parameters and running statistics, and the gradient
// outputs (null: not wanted).
struct BnRef { float *w, *gamma, *beta, *rmean, *rvar; long long* nbt; float *gw, *ggamma, *gbeta; };

// Where a BatchNorm's output goes: y [M pixels, ld] (ld >= C: a channel slice of a wider tensor, e.g. a concat), and
// optionally again into the interior of a [B, H+2, W+2, C] padded buffer (pad; the reflection-padded input of a tensor-core
// conv, whose halo reflect_halo then fills).
struct BnOut { float* y; int ld; float* pad = nullptr; int B = 0, H = 0, W = 0; };

// Train-mode BatchNorm of z [M, C]: per-channel statistics (fp64 sums; running mean / unbiased running var with factor
// momentum, or 1 / num_batches_tracked when momentum < 0; num_batches_tracked += 1, all on the device), then
// y = gamma * (z - mean) * invstd + beta (+ res [M, C]) (ReLU) (TF32-rounded when round).  part: kMaxChunks * C double2.
int bn_forward(const BnRef& r, const float* z, long M, int C, float eps, float momentum, float* mean, float* invstd, const float* res, bool relu,
               bool round, const BnOut& out, double2* part, cudaStream_t st);
// Its backward: g (gradient of y, masked by [y > 0] when y is given) -> gz (may alias g); g_gamma / g_beta into r.ggamma /
// r.gbeta when set.  gb: 2 * C floats of scratch (it holds g_beta, g_gamma).
int bn_backward(const BnRef& r, const float* g, const float* y, const float* z, const float* mean, const float* invstd, long M, int C, bool round,
                float* gz, double2* part, float* gb, cudaStream_t st);
// out[c] = sum over the M rows of x [M, C] (fp64, fixed order): a bias gradient.  part / gb as bn_backward's.
int channel_sum(const float* x, long M, int C, float* out, double2* part, float* gb, cudaStream_t st);

// Split-K chunks of a weight gradient with `tiles` output tiles of `tile_floats` each over M pixels: a function of the
// shape only (fixed summation order), with at most kWgradPart floats of partials.
int wgrad_chunks(long M, long tiles, long tile_floats, long per_chunk_min);
// out[i] = sum_j part[j][i] over n chunks in fixed order (fp64).
int sum_chunks(const float* part, int n, long len, float* out, cudaStream_t st);
// 1x1 weight gradient out[co][ci] = sum over M pixels of g[p][co] * a[p][ci]; part: kWgradPart floats.
int pw_wgrad(const float* g, const float* a, long M, int Co, int Ci, float* part, float* out, cudaStream_t st);

// One weight repacked on the device for smk::conv.  kind MAT: src [rows][cols] -> hi (and lo), transposed when
// `transpose`; split: hi = tf32(v), lo = tf32(v - hi) (lo null: hi only); otherwise hi = v.  The other kinds produce the
// logical matrix W[n][k] of smk::pack_conv3 / the generator's up-convolution (N, K below) in smk::conv's layout: fp32
// [K][N] (split 0), or TF32 [N][K] heads (+ tails in lo) (split 1):
//   CONV3_FWD    torch [cout][cin][3][3]   N = cout,     K = 9 cin_p: W(k = tap cin_p + ci, co) = w[co][ci][tap]
//   CONV3_DGRAD  the same                  N = cin_p,    K = 9 cout:  W'(k = (8 - tap) cout + co, ci) = w[co][ci][tap]
//   UP_FWD       torch [cin][cout][2][2]   N = 4 cout,   K = cin:     W(k = c, n = q cout + o) = w[c][o][q]
//   UP_DGRAD     the same                  N = cin,      K = 4 cout:  W'(k = q cout + o, c) = w[c][o][q]
//   UP_BIAS      bias [cout]               N = 4 cout,   K = 1:       b[n % cout] (split 0)
// Input channels cin..cin_p-1 are zero.
enum PackKind { MAT = 0, CONV3_FWD, CONV3_DGRAD, UP_FWD, UP_DGRAD, UP_BIAS };
struct PackJob { const float* src; float* hi; float* lo; int rows, cols, transpose, split; int kind, cin, cin_p, cout; };
// Floats of a job's output (per copy: lo takes as many again).
size_t pack_floats(const PackJob& j);
// Runs the jobs, as many launches as the job list needs.  bytes: the profiler's byte count of the whole pack.
int pack(const std::vector<PackJob>& jobs, double bytes, cudaStream_t st);

}  // namespace trn
