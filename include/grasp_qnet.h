/* grasp_qnet.h — C-ABI of the batched pixel-wise grasp Q-network forward (libgrasp_qnet.so).
 *
 * Stands in for `policy_net(state)` in the reference agent (Grasping_Agent_multidiscrete.py:254,295) where
 * policy_net = Modules.MULTIDISCRETE_RESNET(6) (Modules.py:308-311).  The layer functions below are the building blocks
 * (one per nn.Module type the network uses); mujoco_rl_ur5_b200/qnet.py strings them together in the order of
 * Perception_Module.forward (Modules.py:170-193) and Grasping_Module_multidiscrete.forward (:256-287).
 * All pointers are CUDA device pointers; activations are NHWC bf16 unless stated; every call is asynchronous on `stream`
 * (cudaStream_t cast to void*).  Return 0 on success, negative on error (gq_last_error()).
 */
#ifndef GRASP_QNET_H
#define GRASP_QNET_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* gq_last_error(void);
const char* gq_version(void);

/* nn.Conv2d(Cin, Cout, kernel_size=ks, padding=ks/2, stride=1) for ks in {1,3}, Cin and Cout multiples of 64 (conv3x3: Modules.py:145-156;
 * BasicBlock.conv3 1x1 with bias: :126).  wgmma implicit GEMM.  x [B,H,W,Cin] bf16, w [Cout][ks*ks][Cin] bf16, bias [Cout] f32 or NULL,
 * y [B,H,W,Cout] f32.  If stats != NULL, stats[B][Cout][2] f32 := per-image (sum, sum of squares) of y over H*W, computed
 * deterministically through `partials`, a scratch buffer of gq_conv_partials_floats(B, H, W, Cout) floats. */
/* size in floats of the `partials` scratch buffer gq_conv_tc needs for per-image statistics: one (sum, sum of squares) row of Cout per
 * consumer warp and 128-pixel tile of every image = B * ceil(H*W/128) * 8 * Cout * 2 */
size_t gq_conv_partials_floats(int B, int H, int W, int Cout);
int gq_conv_tc(const void* x, const void* w, const float* bias, float* y, float* stats, float* partials, int B, int H, int W, int Cin, int Cout, int ks,
               void* stream);
/* Tail of BasicBlock.forward (Modules.py:136-142: `out = bn2(conv2(out)); identity = conv3(x); out += identity; out = relu(out)`) with the
 * shortcut convolution doing the rest in its epilogue: out = relu((resid - mean) * rsqrt(var + eps) * gamma + beta + conv(x, w) + bias) as
 * bf16 [B,H,W,Cout].  resid [B,H,W,Cout] f32 and stats [B,Cout,2] are conv2's outputs from gq_conv_tc; gamma / beta [Cout] are bn2's;
 * scratch_scale_shift: B * Cout * 2 floats.  Same shapes and constraints as gq_conv_tc. */
int gq_conv_tc_block_out(const void* x, const void* w, const float* bias, const float* resid, const float* stats, const float* gamma, const float* beta,
                         float eps, float* scratch_scale_shift, void* out, int B, int H, int W, int Cin, int Cout, int ks, void* stream);
/* Eval-mode BasicBlock convolutions with BatchNorm folded into the weights (BatchNorm2d with running statistics is a per-channel affine map,
 * s = gamma * rsqrt(running_var + eps)): out = [relu](conv_ks_a(a, w[:, :ks_a*ks_a*Ca]) + conv1x1(x, w[:, ks_a*ks_a*Ca:]) + bias) as bf16
 * [B,H,W,Cout], written from the accumulator registers.  a [B,H,W,Ca] bf16; x [B,H,W,Cx] bf16 or NULL (Cx = 0: single source);
 * w [Cout][ks_a*ks_a*Ca + Cx] bf16 (the [Cout][kh][kw][Ca] weights of the first source followed by the [Cout][Cx] 1x1 weights), bias [Cout]
 * f32 or NULL.  Per block (Modules.py:126-142): a1 = relu(conv3x3(x, W1 s1) + beta1 - mu1 s1), then
 * out = relu(conv3x3(a1, W2 s2) + conv1x1(x, W3) + beta2 - mu2 s2 + b3).  Ca, Cx, Cout multiples of 64. */
int gq_conv_tc_fused(const void* a, const void* x, const void* w, const float* bias, void* out, int relu, int B, int H, int W, int Ca, int Cx, int Cout,
                     int ks_a, void* stream);
/* Perception_Module.C1 = conv3x3(4, 64), no bias (Modules.py:163): x [B,4,H,W] f32 NCHW, w [64][3][3][4] f32, y [B,H,W,64] bf16 */
int gq_conv_first(const float* x, const float* w, void* y, int B, int H, int W, void* stream);
/* nn.MaxPool2d(kernel_size=3, stride=2, padding=1) (Modules.py:164,166): x [B,H,W,C] -> y [B,ceil(H/2),ceil(W/2),C] */
int gq_maxpool(const void* x, void* y, int B, int H, int W, int C, void* stream);
/* nn.BatchNorm2d in training mode with per-image statistics + optional residual add + ReLU (BasicBlock.forward, Modules.py:128-142):
 * y = relu((x - mean) * rsqrt(var + eps) * gamma + beta [+ identity]); x, identity [B,HW,C] f32, stats from gq_conv_tc, y bf16 */
int gq_bn_act(const float* x, const float* stats, const float* gamma, const float* beta, const float* identity, void* y, int B, int HW, int C,
              float eps, void* stream);
/* nn.UpsamplingBilinear2d(scale_factor=2) (align_corners=True) (Modules.py:248,250): x [B,H,W,C] -> y [B,2H,2W,C] */
int gq_upsample2x(const void* x, void* y, int B, int H, int W, int C, void* stream);
/* Network tail computed at the lower resolution: Grasping_Module_multidiscrete ends with UP2 -> C1 = nn.Conv2d(64, A, 1) -> squeeze ->
 * Sigmoid (Modules.py:250-251,281-283) and C1 (1x1 conv + bias) commutes with bilinear up-sampling, so q = sigmoid(UP2(C1(x))):
 * x [B,H,W,64] bf16 (the input of UP2), w [A][64] f32, bias [A] f32 (A <= 8), scratch_z [B,A,H,W] f32, q [B,A,2H,2W] f32 (the
 * reference's NCHW output layout) */
int gq_head_up2(const void* x, const float* w, const float* bias, float* scratch_z, float* q, int B, int H, int W, int A, void* stream);
/* Grasp_Agent.transform_observation(normalize=True, jitter_and_noise=False) batched (Grasping_Agent_multidiscrete.py:301-368):
 * rgb [B,HW,3] u8, depth [B,HW] f32 metres -> state [B,4,HW] f32 (rgb/255, depth clipped at depth_threshold, negated, min-max per image);
 * scratch_minmax [B,2] f32 */
int gq_obs_to_state(const unsigned char* rgb, const float* depth, float depth_threshold, float* scratch_minmax, float* state, int B, int HW,
                    void* stream);
/* Grasp_Agent.transform_observation(normalize=True, jitter_and_noise=True) batched - what the agent feeds the network while it learns
 * (Grasping_Agent_multidiscrete.py:118-124 ColorJitter(0.5, 0.5, 0.5, 0.5), :318 depth += N(0, 0.001) before the min-max normalisation).
 * noise_std: standard deviation of the depth noise (0.001); seed / env_index [B] int64 (NULL: 0..B-1) / step: key and counter of the
 * counter-based generator, so a pixel's noise depends on (seed, global env id, step, pixel) only; jitter [B,4] f32 = brightness,
 * contrast, saturation, hue factors and order [B,4] int32 = the permutation of the four operations, both drawn by the caller as
 * torchvision's ColorJitter.get_params does (NULL jitter: no colour change; NULL order: 0,1,2,3); scratch_red [B,4] f32.
 * Outputs (either may be NULL): state [B,4,HW] f32 (the agent's tensor layout), state_nhwc_bf16 [B,HW,4] bf16 (NHWC, feeds the first
 * convolution without a repack). */
int gq_obs_to_state_train(const unsigned char* rgb, const float* depth, float depth_threshold, float noise_std, unsigned long long seed,
                          const long long* env_index, unsigned int step, const float* jitter, const int* order, float* scratch_red, float* state,
                          void* state_nhwc_bf16, int B, int HW, void* stream);
/* The same training transform with every random choice keyed, for the online trainer and its observation replay.  Row b of the output
 * is image slot[b] of rgb [S,HW,3] u8 / depth [S,HW] f32 (slot [B] int64, NULL: b), keyed on env_index[b] (int64, the global env id)
 * and step[b] (uint32): the depth noise as in gq_obs_to_state_train, and the ColorJitter factors and operation order drawn from the
 * same generator (the table in csrc/qnet.cu), so the state of a stored observation is regenerated bit for bit.
 * Out: jitter_out [B,4] f32 and order_out [B,4] int32 = the drawn factors and order (what gq_obs_to_state_train would be given);
 * state [B,4,HW] f32 and/or state_nhwc_bf16 [B,HW,4] bf16 (either may be NULL); scratch_red [B,4] f32. */
int gq_obs_to_state_keyed(const unsigned char* rgb, const float* depth, const long long* slot, const long long* env_index, const unsigned int* step,
                          float depth_threshold, float noise_std, unsigned long long seed, float* scratch_red, float* jitter_out, int* order_out,
                          float* state, void* state_nhwc_bf16, int B, int HW, void* stream);
/* Grasp_Agent.epsilon_greedy (Grasping_Agent_multidiscrete.py:232-282) for B envs.  depth [B,H,W] f32 (the current observation),
 * greedy_idx [B] int32 (gq_argmax), eps [B] f64, env_index [B] int64 (global env ids), seed / step: key and counter of the keyed draws.
 * Env b is greedy iff its uniform u > eps[b]; otherwise it takes the first of its candidates (flat rot*H*W + y*W + x) whose pixel lies
 * on or above z_min in the world (TABLE_HEIGHT - 0.01), with pixel_2_world's arithmetic for the camera (fovy, cam_pos[3], cam_mat[9]:
 * plain host doubles, the camera of the scene arrays).  After max_draws rejected candidates the last one is taken and exhausted[b] = 1.
 * Out: action [B,2] int32 (pixel y*W + x, rotation), is_random [B] u8, exhausted [B] u8. */
int gq_sample_actions(const float* depth, const int* greedy_idx, const double* eps, unsigned long long seed, const long long* env_index, unsigned int step,
                      double fovy, const double* cam_pos, const double* cam_mat, double z_min, int W, int H, int R, int max_draws, int B, int* action,
                      unsigned char* is_random, unsigned char* exhausted, void* stream);
/* output.view(-1).max(0) per image (Grasping_Agent_multidiscrete.py:295-299): q [B,n] -> idx [B] int32 (rot*HW + y*W + x), val [B] f32 */
int gq_argmax(const float* q, int B, int n, int* idx, float* val, void* stream);
/* The Bellman target of the bootstrapped learn() (Grasping_Agent_multidiscrete.py:430-437: q_expected = reward + GAMMA *
 * target_net(next_state).max(1)[0]) from the target network's head input, without the Q-map: x [B,H,W,64] bf16, w [A][64] f32,
 * bias [A] f32 (A <= 8) as for gq_head_up2, reward [B] f32.  Out: qmax [B] f32 = the largest of the [A,2H,2W] sigmoids of each image,
 * bit for bit the val of gq_argmax on the q of gq_head_up2; y [B] f32 = min(1, reward + gamma * qmax), product and sum each rounded to
 * fp32 (no FMA), so that y stays in binary_cross_entropy's [0, 1] and equals reward at gamma = 0.  Deterministic. */
int gq_head_max_target(const void* x, const float* w, const float* bias, const float* reward, float gamma, float* qmax, float* y, int B, int H, int W,
                       int A, void* stream);

/* ------------------------------------------------------------------------------------------------------------------------------------
 * Learner: the compute of Grasp_Agent.learn() (Grasping_Agent_multidiscrete.py:388-446, optimiser :153-156) - see csrc/qnet_learn.cuh.
 * All buffers [dev]; activations NHWC bf16, pre-BatchNorm outputs fp32, gradients of activations bf16, of parameters fp32. */
/* BatchNorm over the whole batch (learn() forwards B images at once, training mode): per-image sums -> batch sums, in place.
 * stats [B,C,2] as written by gq_conv_tc. */
int gq_bn_batch_merge(float* stats, int B, int C, void* stream);
/* nn.BatchNorm2d's running-statistics update in a training-mode forward (torch's _BatchNorm.forward with momentum 0.1; the reference's
 * policy_net(state_batch) in train mode, Grasping_Agent_multidiscrete.py:426 and Offline RL/train.py:109):
 *   r_mean = (1 - m) r_mean + m mean,  r_var = (1 - m) r_var + m var n / (n - 1),  n = B*HW,
 * with mean = s1 / HW, var = s2 / HW - mean^2 from merged_stats [B,C,2] as gq_bn_batch_merge leaves them (row 0 is read).  Double
 * arithmetic, one thread per channel.  running_mean / running_var [C] f32, updated in place. */
int gq_bn_running_update(const float* merged_stats, float* running_mean, float* running_var, int B, int HW, int C, float momentum, void* stream);
/* q_pred = net(state).view(B,-1).gather(1, action); loss = binary_cross_entropy(q_pred, reward) (Grasping_Agent_multidiscrete.py:426-443)
 * + backward through sigmoid, the bilinear 2x up-sampling of the head planes and the 1x1 head convolution (Modules.py:250-251,281-283):
 * q [B,A,2H,2W] f32 (forward output), x [B,H,W,64] bf16 (head input), w_head [A,64] f32, action [B] int64 (rot*4HW + y*2W + x), reward [B] f32.
 * Out: loss_terms [B] (mean = the loss), qsel [B] = q_pred, dX [B,H,W,64] bf16, dW_head [A,64], db_head [A]; partials [B,A,64], [B,A].
 * As in torch's fp32 autograd, an image whose q_pred is exactly 0 or 1 contributes loss 100 (or 0) and no gradient. */
int gq_loss_head_bwd(const float* q, const void* x, const float* w_head, const long long* action, const float* reward, int B, int A, int H, int W,
                     float* loss_terms, float* qsel, void* dX, float* dW_partial, float* db_partial, float* dW_head, float* db_head, void* stream);
/* The same with importance weights weight [B] f32 (prioritized replay): loss = mean(w_b loss_b) = binary_cross_entropy(q_pred, reward,
 * weight=w), loss_terms[b] = w_b loss_b and the gradient of image b scaled by w_b.  With every w_b = 1 the outputs equal gq_loss_head_bwd's
 * bit for bit. */
int gq_loss_head_bwd_weighted(const float* q, const void* x, const float* w_head, const long long* action, const float* reward, const float* weight, int B,
                              int A, int H, int W, float* loss_terms, float* qsel, void* dX, float* dW_partial, float* db_partial, float* dW_head,
                              float* db_head, void* stream);
/* backward of y = relu(BatchNorm(o) [+ identity]) with batch statistics (BasicBlock, Modules.py:128-142): dY, act = y [B,HW,C] bf16, o [B,HW,C] f32,
 * stats merged [B,C,2], gamma [C], C a multiple of 8.  Out: d_o [B,HW,C] bf16 (gradient w.r.t. the convolution output), dgamma, dbeta [C] (either may be NULL),
 * dpre_out (NULL or [B,HW,C] bf16) = dY * (y > 0), the gradient that also enters the identity branch.
 * scratch_part: ceil(B*HW/128) * C * 2 floats, scratch_sums: 2 C floats. */
int gq_bn_relu_bwd(const void* dY, const void* act, const float* o, const float* stats, const float* gamma, int B, int HW, int C, float eps,
                   void* dpre_out, float* scratch_part, float* scratch_sums, float* dgamma, float* dbeta, void* d_o, void* stream);
/* weight gradient of conv3x3 / conv1x1 (Modules.py:145-156): dY [B,H,W,Cout] bf16, x [B,H,W,Cin] bf16 -> dW [Cout][ks*ks][Cin] f32;
 * scratch_part: B * Cout * ks*ks * Cin floats (split-K over the images, reduced in image order) */
int gq_conv_wgrad(const void* dY, const void* x, float* scratch_part, float* dW, int B, int H, int W, int Cin, int Cout, int ks, void* stream);
/* weight gradient of Perception_Module.C1 (4 -> 64, Modules.py:163): dY [B,H,W,64] bf16, x [B,4,H,W] f32 -> dW [64][3][3][4] f32;
 * scratch_part: ceil(B*H*W/2048) * 64 * 36 floats */
int gq_conv_first_wgrad(const void* dY, const float* x, float* scratch_part, float* dW, int B, int H, int W, void* stream);
/* MaxPool2d(3, 2, 1) backward: x [B,H,W,C] bf16 (pool input), dY [B,ceil(H/2),ceil(W/2),C] bf16 -> dX [B,H,W,C] bf16; C a multiple of 8 */
int gq_maxpool_bwd(const void* x, const void* dY, void* dX, int B, int H, int W, int C, void* stream);
/* UpsamplingBilinear2d(2) backward: dY [B,2H,2W,C] bf16 -> dX [B,H,W,C] bf16 */
int gq_upsample2x_bwd(const void* dY, void* dX, int B, int H, int W, int C, void* stream);
/* out (bf16) = a (f32) + b (f32, may be NULL) or a + c_bf16 (bf16, may be NULL): sums two gradient branches */
int gq_add_to_bf16(const float* a, const float* b, const void* c_bf16, void* out, size_t n, void* stream);
/* torch.optim.Adam step with weight_decay as L2 (Grasping_Agent_multidiscrete.py:153-156): p, g, m, v [n] f32, step counted from 1 */
int gq_adam(float* p, const float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps, float weight_decay, int step, void* stream);
/* torch.optim.SGD step with dampening 0 and nesterov off (Grasping_Agent_multidiscrete.py:145-152, momentum 0.9, weight_decay 2e-5):
 * d = g + wd p; buf = d when `first` (the buffer's first step), else momentum buf + d; p -= lr buf.  p, g, buf [n] f32; with momentum 0
 * there is no buffer (buf may be NULL) and p -= lr d.  Each product and sum is rounded separately (no FMA contraction). */
int gq_sgd(float* p, const float* g, float* buf, size_t n, float lr, float momentum, float weight_decay, int first, void* stream);
/* gradient accumulation over micro-batches: acc = g when `first`, else acc + g (fp32, [n]) */
int gq_grad_accumulate(float* acc, const float* g, size_t n, int first, void* stream);

/* ------------------------------------------------------------------------------------------------------------------------------------
 * Prioritized experience replay (Schaul et al. 2016, proportional) - see csrc/qnet_replay.cuh.  tree [2 cap] f64: an implicit sum-tree,
 * cap = the smallest power of two >= the replay size (at most 2^30), slot i = leaf cap + i, node k = tree[2k] + tree[2k+1], root
 * tree[1]; zero-initialised by the caller.  pmax [1] f64 = the largest priority ever assigned, 1.0 initially. */
/* new transitions: leaves of slot [n] int64 (distinct, < cap) := pmax, ancestors recomputed */
int gq_per_push(double* tree, const double* pmax, const long long* slot, int n, int cap, void* stream);
/* stratified proportional sampling of B <= 1024 slots: stratum j draws U from Philox4x32-10 (counter (0xC0000000 + j, update_lo, update_hi,
 * rank), key (seed_lo, seed_hi)), u = (j + U) total / B, and descends from the root (right iff u >= left and the right sum > 0).
 * length = slots filled (the N of the weights).  Out: idx_out [B] int64, weight_out [B] f32 = (length p_j / total)^-beta / max_j(...) */
int gq_per_sample(const double* tree, int cap, long long length, int B, double beta, unsigned long long seed, unsigned long long update, unsigned int rank,
                  long long* idx_out, float* weight_out, void* stream);
/* priorities of a trained batch: p_j = (|reward_j - qsel_j| + eps)^alpha, applied in batch order (a slot drawn twice keeps the later value),
 * ancestors recomputed, pmax raised.  idx [B] int64 (B <= 1024), qsel / reward [B] f32 */
int gq_per_update(double* tree, double* pmax, const long long* idx, const float* qsel, const float* reward, int B, double alpha, double eps, int cap,
                  void* stream);

#ifdef __cplusplus
}
#endif
#endif
