// The generator's backward building blocks (generator.cu), shared by the input gradient of the eval path and the train path
// (generator_train.cu).  NHWC fp32 activations; `round` rounds the result to TF32 for a TF32 consumer.
#pragma once
#include "conv.cuh"

// fwd / dgrad: the weight operands of the forward and of the input gradient (smk::pack_conv3; the dgrad's carry the BN scale)
struct Conv3 { smk::GemmW fwd, dgrad; float* scale; float* bias; int cin, cin_p, cout; };
// fwd: N = 4*cout (n = (dy*2+dx) * cout + co), K = cin; dgrad: N = cin, K = 4*cout
struct UpConv { smk::GemmW fwd, dgrad; float* scale; float* bias; int cin, cout; };

namespace gen {

// A train handle's topology (generator_train.cu).  t: index of the layer's first tensor in the tensor list (state_dict
// order without num_batches_tracked: a 3x3 conv's weight, then its BatchNorm's weight, bias, running_mean, running_var);
// bn: the BatchNorm's index (num_batches_tracked); sv_z / sv_y: saved indices of the conv's pre-BN output and of the
// BatchNorm's (+ residual) (+ ReLU) output (-1: stored elsewhere); stats: float offset of mean[cout] (invstd[cout] follows)
// in the statistics after the saved tensors.
struct TrainConv { int t = 0, bn = 0, cin = 0, cin_p = 0, cout = 0, S = 0; bool refl = false; int sv_z = -1, sv_y = -1; size_t stats = 0; };
struct TrainUp { int t = 0, cin = 0, cout = 0; };
struct TrainTopo {
    TrainConv enc[5][2], dec[4][2];          // encoder1..4, bottleneck; decoder4..1
    std::vector<TrainConv> res;              // 2 per ResnetBlock
    TrainUp up[4];                           // upconv4..1
    int head_t = 0, n_tensors = 0, n_bn = 0;
    int sv_input = -1, sv_cat[4] = {-1, -1, -1, -1}, sv_pool[4] = {-1, -1, -1, -1};   // cat / pool: index 0 = 224^2
    size_t stats_floats = 0;
};

}  // namespace gen

struct SmkGenerator {
    int cin, cin_p, cout, f, nres, precision;
    Conv3 enc[5][2];                 // encoder1..4, bottleneck
    std::vector<Conv3> res;          // 2 per ResnetBlock
    UpConv up[4];                    // upconv4..1  (index 0 = level 4)
    Conv3 dec[4][2];                 // decoder4..1
    float *fw = nullptr, *fb = nullptr;   // final 1x1: W[f][cout], bias
    float *ones = nullptr, *zeros = nullptr;   // unit scale / zero bias of the dgrad epilogues
    smk::SavedLayout saved;          // activations of the grad-mode forward, forward order
    smk::DeviceArena arena;
    bool train = false;              // a train handle (smk_generator_train_create): topology only, no packed weights
    gen::TrainTopo topo;             // train handles
};

namespace gen {

// dgrad of a 3x3 conv (zero padding 1) over S x S: out = conv3x3(g, W') * [mask > 0] (mask null: none), W' the packed dgrad
// operand (N = cin_p, K = 9 cout, see smk::pack_conv3); ones / zeros: >= cin_p unit scales / zero biases.
int dgrad3(const smk::GemmW& w, int cin_p, int cout, const float* ones, const float* zeros, const float* g, int B, int S, const float* mask,
           float* out, int ld_out, bool round, cudaStream_t st);
// dgrad of ConvTranspose2d(k2, s2): out [S x S, cin] = s2d [S x S, 4 cout] . W'^T * [mask > 0], W' packed with N = cin, K = 4 cout.
int dgrad_up(const smk::GemmW& w, int cin, int cout, const float* ones, const float* zeros, const float* s2d, int B, int S, const float* mask,
             float* out, bool round, cudaStream_t st);
// Space-to-depth of the up-convolution's output gradient (C of the ld_in channels): out[b,h,w,(dy*2+dx)*C + c] =
// in[b,2h+dy,2w+dx,c], S the output size.
int s2d(const float* in, int ld_in, int B, int S, int C, float* out, cudaStream_t st);
// Adjoint of ReflectionPad2d(1) at 14 x 14: out = (fold(gP) + res) * [mask > 0], each term optional (see fold_kernel);
// out_pad: write [B,16,16,C] with a zero halo.
int fold(const float* gP, const float* res, int res_pad, const float* mask, int B, int C, bool round, float* out, int out_pad, cudaStream_t st);
// MaxPool 2x2 backward + skip gradient + ReLU mask of the pool input e [B,S,S,C] (pixel stride ld_e):
// out = (g_skip + [first maximum of the window] * g_p) * [e > 0], [B,S,S,C].
int pool_bwd(const float* e, int ld_e, const float* gp, const float* gskip, int ld_skip, int B, int S, int C, bool round, float* out, cudaStream_t st);
// Head: out[b,p,c] = (sum_j W_h[c][j] * g_y[b,j,p] * y (1 - y)) * [d > 0], NCHW g_y / y -> NHWC [B,HW,f]; W_h [f][cout].
int head_bwd(const float* gy, const float* y, int B, int HW, int cout, const float* w, const float* d, int f, bool round, float* out, cudaStream_t st);
// First C of Cp channels, NHWC [B,HW,Cp] -> NCHW [B,C,HW].
int nhwc_to_nchw(const float* in, int B, int HW, int Cp, int C, float* out, cudaStream_t st);

}  // namespace gen
