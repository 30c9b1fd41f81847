// Backward pass + optimiser of the pixel-wise grasp Q-network: the compute of Grasp_Agent.learn()
// (reference: Grasping_Agent_multidiscrete.py:388-446; optimiser :153-156 Adam(lr, weight_decay 2e-5); network Modules.py:92-311).
//
//   q_pred = policy_net(state_batch).view(B, -1).gather(1, action_batch);  loss = binary_cross_entropy(q_pred, reward);  loss.backward();
//   optimizer.step()
//
// In learn() the network sees the whole batch, so BatchNorm (training mode) normalises over batch AND pixels - unlike the acting
// forward, which runs one image at a time (per-image statistics).  gq_bn_batch_merge turns the per-image sums the convolution
// epilogue produces into batch sums, after which the forward kernels of qnet.cu compute exactly that.
//
// Data layout as in the forward: activations NHWC bf16, pre-BatchNorm convolution outputs fp32, weights [Cout][kh][kw][Cin].
// Gradients of activations travel as bf16 between layers (fp32 inside a kernel), weight gradients and the optimiser state are fp32.
//   dgrad (gradient w.r.t. the convolution input) = the forward wgmma convolution applied to dY with the spatially flipped,
//          in/out-transposed weights (gq_conv_tc called by the host wrapper);
//   wgrad (gradient w.r.t. the weights)           = k_wgrad_wgmma below: wgmma GEMM with K = pixels, both operands MN-major straight from the
//          NHWC tensors by TMA, split-K over the images of the batch (partials reduced in image order: deterministic);
//   everything else is element-wise / reduction glue.
// Included at the end of qnet.cu (same library, C-ABI in include/grasp_qnet.h).
#pragma once

// ------------------------------------------------------------------------------------------------ BatchNorm over the batch
// stats [B,C,2] per-image (sum, sum of squares) -> every image's entry := batch total / B, so that the per-image formulas
// mean = s1 / HW, var = s2 / HW - mean^2 of k_bn_act / k_bn_scale_shift yield the statistics over B * HW values
__global__ void k_bn_batch_merge(float* __restrict__ stats, int B, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s1 = 0, s2 = 0;
  for (int b = 0; b < B; b++) { s1 += stats[((size_t)b * C + c) * 2]; s2 += stats[((size_t)b * C + c) * 2 + 1]; }
  const float m1 = (float)(s1 / B), m2 = (float)(s2 / B);
  for (int b = 0; b < B; b++) { stats[((size_t)b * C + c) * 2] = m1; stats[((size_t)b * C + c) * 2 + 1] = m2; }
}
// nn.BatchNorm2d's running-statistics update of a training-mode forward (momentum m): from the merged stats (row 0 = batch average of
// the per-image sums) the batch mean and biased variance the forward normalises with, then r_mean = (1-m) r_mean + m mean and
// r_var = (1-m) r_var + m var n/(n-1) with n = B*HW values per channel (torch stores the unbiased variance).  One thread per channel.
__global__ void k_bn_running_update(const float* __restrict__ stats, float* __restrict__ rmean, float* __restrict__ rvar, int C, double HW, double n,
                                    double m) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double mean = (double)stats[(size_t)c * 2] / HW, var = fmax((double)stats[(size_t)c * 2 + 1] / HW - mean * mean, 0.0);
  rmean[c] = (float)((1.0 - m) * (double)rmean[c] + m * mean);
  rvar[c] = (float)((1.0 - m) * (double)rvar[c] + m * var * n / (n - 1.0));
}

// ------------------------------------------------------------------------------------------------ loss + head backward
// One CTA per image.  q [B,A,2H,2W] (sigmoid of the bilinearly up-sampled head output), x [B,H,W,64] bf16 (input of the head),
// action [B] = rot * (2H*2W) + y * 2W + x, reward [B].  With v = pre-sigmoid value at the chosen pixel, dL/dv follows torch's chain
// rule in fp32: BCE backward (q - r) / B / max(q (1 - q), 1e-12), then the sigmoid's q (1 - q).  Mathematically that is (q - r) / B, but
// where q rounds to exactly 1 or 0 (logit above ~16.6 or below ~-88) torch's gradient is 0 (the loss is clamped at 100), and so is this one.
// v = UP2(z)[rot, y, x] = sum of 4 bilinear taps of z = W_head x + b on the H x W map, so the gradient reaches 4 (or fewer) pixels:
//   dx[pix,:] += g w W_head[rot,:],  dW_head[rot,:] += g w x[pix,:],  db_head[rot] += g w.
// Outputs: loss_terms [B] (-(r log q + (1-r) log(1-q)), logs clamped at -100 like torch), dX [B,H,W,64] bf16 (zero-filled by the
// caller, 4 rows written here), dWp [B,A,64] / dbp [B,A] per-image partials (zero except row rot), qsel [B] the gathered q.
// weight [B] (NULL: every w_b = 1, the unweighted loss bit for bit): importance weights of prioritized replay, the loss
// mean(w_b loss_b) = binary_cross_entropy(q, r, weight=w); loss_terms[b] and the gradient of image b are scaled by w_b.
__global__ void __launch_bounds__(64) k_loss_head_bwd(const float* __restrict__ q, const bf16* __restrict__ x, const float* __restrict__ w_head,
                                                     const long long* __restrict__ action, const float* __restrict__ reward, const float* __restrict__ weight,
                                                     int B, int A, int H, int W, float* __restrict__ loss_terms, float* __restrict__ qsel, bf16* __restrict__ dX, float* __restrict__ dWp,
                                                     float* __restrict__ dbp) {
  const int b = blockIdx.x, c = threadIdx.x;  // thread = head input channel
  const int OH = 2 * H, OW = 2 * W;
  const long long a = action[b];
  const int rot = (int)(a / ((long long)OH * OW)), oy = (int)((a / OW) % OH), ox = (int)(a % OW);
  const float qv = q[(((size_t)b * A + rot) * OH + oy) * OW + ox], r = reward[b];
  const float wb = weight ? weight[b] : 1.f;
  if (c == 0) {
    const float term = -(r * fmaxf(logf(qv), -100.f) + (1.f - r) * fmaxf(logf(1.f - qv), -100.f));
    loss_terms[b] = weight ? wb * term : term;
    qsel[b] = qv;
  }
  const float sg = (1.f - qv) * qv;
  const float g = (wb / (float)B) * (qv - r) / fmaxf(sg, 1e-12f) * sg;
  const float fy = oy * (float)(H - 1) / (float)(OH - 1), fx = ox * (float)(W - 1) / (float)(OW - 1);
  const int y0 = (int)fy, x0 = (int)fx, y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  const float wy = fy - y0, wx = fx - x0;
  const int py[4] = {y0, y0, y1, y1}, px[4] = {x0, x1, x0, x1};
  const float wt[4] = {(1 - wx) * (1 - wy), wx * (1 - wy), (1 - wx) * wy, wx * wy};
  for (int aa = 0; aa < A; aa++) dWp[((size_t)b * A + aa) * 64 + c] = 0.f;
  if (c < A) dbp[(size_t)b * A + c] = 0.f;
  __syncthreads();
  const float wh = w_head[rot * 64 + c];
  float dw = 0.f, db = 0.f;
  // coincident taps (image border) are merged first so that a pixel row is written once
  float acc[4] = {wt[0], wt[1], wt[2], wt[3]};
  bool live[4] = {true, true, true, true};
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < i; j++)
      if (live[i] && live[j] && py[i] == py[j] && px[i] == px[j]) { acc[j] += acc[i]; live[i] = false; }
  for (int i = 0; i < 4; i++) {
    if (!live[i]) continue;
    const size_t pix = ((size_t)b * H + py[i]) * W + px[i];
    const float xv = __bfloat162float(x[pix * 64 + c]);
    dw += g * acc[i] * xv;
    db += g * acc[i];
    dX[pix * 64 + c] = __float2bfloat16(g * acc[i] * wh);
  }
  dWp[((size_t)b * A + rot) * 64 + c] = dw;
  if (c == 0) dbp[(size_t)b * A + rot] = db;
}

// out[n] = sum over rows r < R of part[r][n], in row order (deterministic); used for per-image partials and split-K partials
__global__ void k_reduce_rows(const float* __restrict__ part, float* __restrict__ out, int R, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int r = 0; r < R; r++) s += part[(size_t)r * n + i];
  out[i] = s;
}

// ------------------------------------------------------------------------------------------------ BatchNorm (+ReLU) backward
// Layer: y = relu(gamma * xhat + beta [+ identity]),  xhat = (o - mean) * rstd with batch statistics (from the merged stats).
// dY [B*HW, C] bf16 gradient w.r.t. y, act [B*HW, C] bf16 = y (ReLU mask: y > 0), o [B*HW, C] fp32 pre-BN convolution output.
// Pass 1 (k_bn_bwd_reduce): per CTA (a block of rows) and channel: sum dpre, sum dpre * xhat, with dpre = dY * (y > 0); optionally
//         writes dpre as bf16 (the gradient that also flows into the shortcut convolution / the identity branch).
// Pass 2 (k_bn_bwd_apply8): d_o = gamma * rstd * (dpre - S1 / N - xhat * S2 / N) as bf16;  dgamma = S2, dbeta = S1.
__global__ void __launch_bounds__(256) k_bn_bwd_reduce(const bf16* __restrict__ dY, const bf16* __restrict__ act, const float* __restrict__ o,
                                                       const float* __restrict__ stats, int rows, int C, int HW, float eps, int rows_per_cta,
                                                       bf16* __restrict__ dpre_out, float* __restrict__ part) {
  // 256 threads = Cw channels x RL row lanes (Cw = min(C, 256)): consecutive threads read consecutive channels of a row (coalesced), row lane
  // rl takes rows r0 + rl, r0 + rl + RL, ...; the row lanes are added in fixed order through shared memory.  (With one thread per
  // channel only 64 / 128 of the 256 threads would work in the 64- / 128-channel layers.)
  __shared__ float sh[2][256];
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  for (int cb = 0; cb < C; cb += 256) {
    const int Cw = min(C - cb, 256), RL = 256 / Cw, c = cb + (int)threadIdx.x % Cw, rl = (int)threadIdx.x / Cw;
    float a1 = 0.f, a2 = 0.f;
    if (rl < RL) {
      const float s1 = stats[(size_t)c * 2], s2 = stats[(size_t)c * 2 + 1];  // image 0's entry = batch value after the merge
      const float mean = s1 / HW, var = fmaxf(s2 / HW - mean * mean, 0.f), rstd = rsqrtf(var + eps);
      for (int r = r0 + rl; r < r1; r += RL) {
        const size_t i = (size_t)r * C + c;
        const float d = __bfloat162float(act[i]) > 0.f ? __bfloat162float(dY[i]) : 0.f;
        if (dpre_out) dpre_out[i] = __float2bfloat16(d);
        a1 += d;
        a2 += d * ((o[i] - mean) * rstd);
      }
    }
    sh[0][threadIdx.x] = a1; sh[1][threadIdx.x] = a2;
    __syncthreads();
    if ((int)threadIdx.x < Cw) {
      float t1 = 0.f, t2 = 0.f;
      for (int k = 0; k < RL; k++) { t1 += sh[0][k * Cw + threadIdx.x]; t2 += sh[1][k * Cw + threadIdx.x]; }
      part[((size_t)blockIdx.x * C + cb + threadIdx.x) * 2] = t1;
      part[((size_t)blockIdx.x * C + cb + threadIdx.x) * 2 + 1] = t2;
    }
    __syncthreads();
  }
}
// sums[C,2] = per-channel totals of the partials; dgamma[c] = sums[c][1], dbeta[c] = sums[c][0].  One warp per channel: lane l adds parts
// l, l + 32, ... in order, then a fixed butterfly over the lanes (deterministic; one thread per channel would walk ~1000 partials
// alone).
__global__ void __launch_bounds__(128) k_bn_bwd_sums(const float* __restrict__ part, int nparts, int C, float* __restrict__ sums, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= C) return;
  double a1 = 0, a2 = 0;
  for (int k = lane; k < nparts; k += 32) { a1 += part[((size_t)k * C + c) * 2]; a2 += part[((size_t)k * C + c) * 2 + 1]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a1 += __shfl_xor_sync(0xffffffffu, a1, o); a2 += __shfl_xor_sync(0xffffffffu, a2, o); }
  if (lane == 0) {
    sums[c * 2] = (float)a1; sums[c * 2 + 1] = (float)a2;
    if (dgamma) dgamma[c] = (float)a2;
    if (dbeta) dbeta[c] = (float)a1;
  }
}
// pass 2, 8 consecutive channels per thread (16-byte loads / stores; C % 8 == 0)
__global__ void __launch_bounds__(256) k_bn_bwd_apply8(const bf16* __restrict__ dY, const bf16* __restrict__ act, const float* __restrict__ o,
                                                       const float* __restrict__ stats, const float* __restrict__ gamma, const float* __restrict__ sums,
                                                       size_t n8, int C, int HW, float invN, float eps, bf16* __restrict__ d_o) {
  size_t i8 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i8 >= n8) return;
  const size_t i = i8 * 8;
  const int c0 = (int)(i % C);
  const uint4 qd = *(const uint4*)(dY + i), qa = *(const uint4*)(act + i);
  const float4 o0 = *(const float4*)(o + i), o1 = *(const float4*)(o + i + 4);
  const float ov[8] = {o0.x, o0.y, o0.z, o0.w, o1.x, o1.y, o1.z, o1.w};
  const __nv_bfloat162 *pd = (const __nv_bfloat162*)&qd, *pa = (const __nv_bfloat162*)&qa;
  __nv_bfloat162 out[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float2 fd = __bfloat1622float2(pd[k]), fa = __bfloat1622float2(pa[k]);
    float r[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int c = c0 + 2 * k + h;
      const float s1 = stats[(size_t)c * 2], s2 = stats[(size_t)c * 2 + 1];
      const float mean = s1 / HW, var = fmaxf(s2 / HW - mean * mean, 0.f), rstd = rsqrtf(var + eps);
      const float xhat = (ov[2 * k + h] - mean) * rstd;
      const float d = (h ? fa.y : fa.x) > 0.f ? (h ? fd.y : fd.x) : 0.f;
      r[h] = gamma[c] * rstd * (d - sums[c * 2] * invN - xhat * sums[c * 2 + 1] * invN);
    }
    out[k] = __floats2bfloat162_rn(r[0], r[1]);
  }
  *(uint4*)(d_o + i) = *(const uint4*)out;
}

// first convolution (4 -> 64 channels, 3x3, no bias; Modules.py:163): dW[co][tap][c] = sum_{b,p} dY[b,p,co] * x[b,c,p+tap] with x the
// network input [B,4,H,W] f32.  One CTA = one chunk of pixels for ALL 36 (tap, c) pairs: thread (co, quarter) walks a quarter of the
// chunk with 36 accumulators (dY read once; the 36 input values of a pixel are the same for all threads = broadcast loads), the four
// quarters are added in fixed order -> part [chunks][64][36].  (One CTA of 64 threads per (tap, c, chunk) would read dY 36 times.)
__global__ void __launch_bounds__(256) k_conv_first_wgrad(const bf16* __restrict__ dY, const float* __restrict__ x, float* __restrict__ part, int B, int H, int W,
                                                          int pix_per_cta) {
  __shared__ float red[4][64][37];
  const int co = threadIdx.x & 63, q = threadIdx.x >> 6, HW = H * W, quarter = pix_per_cta / 4;
  const long long n = (long long)B * HW, c0 = (long long)blockIdx.x * pix_per_cta + (long long)q * quarter;
  const int i0 = (int)(c0 < n ? c0 : n), i1 = (int)(c0 + quarter < n ? c0 + quarter : n);  // (B * H * W < 2^31: checked by the caller)
  float acc[36];
#pragma unroll
  for (int j = 0; j < 36; j++) acc[j] = 0.f;
  int b = i0 / HW, p = i0 - b * HW, oh = p / W, ow = p - oh * W;  // walked incrementally: no division in the loop
  const bf16* dp = dY + (size_t)i0 * 64 + co;
  for (int i = i0; i < i1; i++, dp += 64) {
    const float d = __bfloat162float(*dp);
    const float* xb = x + (size_t)b * 4 * HW;
#pragma unroll
    for (int tap = 0; tap < 9; tap++) {
      const int ih = oh + tap / 3 - 1, iw = ow + tap % 3 - 1;
      if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
      const float* xp = xb + ih * W + iw;
#pragma unroll
      for (int c = 0; c < 4; c++) acc[tap * 4 + c] += d * __ldg(xp + c * HW);
    }
    if (++ow == W) { ow = 0; if (++oh == H) { oh = 0; b++; } }
  }
#pragma unroll
  for (int j = 0; j < 36; j++) red[q][co][j] = acc[j];
  __syncthreads();
  for (int idx = threadIdx.x; idx < 64 * 36; idx += 256) {
    const int c2 = idx / 36, j = idx % 36;
    part[((size_t)blockIdx.x * 64 + c2) * 36 + j] = ((red[0][c2][j] + red[1][c2][j]) + red[2][c2][j]) + red[3][c2][j];
  }
}

// ------------------------------------------------------------------------------------------------ pooling / up-sampling backward, glue
// MaxPool2d(3, stride 2, padding 1) backward in gather form: input pixel (ih, iw) receives dY of every window whose arg-max it is
// (first maximum in window scan order, as PyTorch does).  x [B,H,W,C] bf16 (the pool's input), dY [B,OH,OW,C] bf16 -> dX [B,H,W,C] bf16;
// 8 channels per thread (16-byte loads; C % 8 == 0)
__global__ void __launch_bounds__(256) k_maxpool_bwd8(const bf16* __restrict__ x, const bf16* __restrict__ dY, bf16* __restrict__ dX, int B, int H, int W, int C) {
  const int OH = (H + 1) / 2, OW = (W + 1) / 2, C8 = C / 8;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)B * H * W * C8;
  if (i >= n) return;
  const int c8 = (int)(i % C8), iw = (int)((i / C8) % W), ih = (int)((i / ((size_t)C8 * W)) % H), b = (int)(i / ((size_t)C8 * W * H));
  float g[8];
#pragma unroll
  for (int k = 0; k < 8; k++) g[k] = 0.f;
  for (int oh = ih / 2; oh <= (ih + 1) / 2 && oh < OH; oh++)
    for (int ow = iw / 2; ow <= (iw + 1) / 2 && ow < OW; ow++) {
      float best[8]; int bpos[8];
#pragma unroll
      for (int k = 0; k < 8; k++) { best[k] = -3.0e38f; bpos[k] = -1; }
      for (int kh = 0; kh < 3; kh++)
        for (int kw = 0; kw < 3; kw++) {
          const int hh = oh * 2 - 1 + kh, ww = ow * 2 - 1 + kw;
          if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
          const uint4 q = *(const uint4*)(x + (((size_t)b * H + hh) * W + ww) * C + c8 * 8);
          const __nv_bfloat162* p2 = (const __nv_bfloat162*)&q;
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const float2 f = __bfloat1622float2(p2[k]);
            if (f.x > best[2 * k]) { best[2 * k] = f.x; bpos[2 * k] = kh * 3 + kw; }
            if (f.y > best[2 * k + 1]) { best[2 * k + 1] = f.y; bpos[2 * k + 1] = kh * 3 + kw; }
          }
        }
      const int mine = (ih - (oh * 2 - 1)) * 3 + (iw - (ow * 2 - 1));  // where (ih, iw) sits in this window
      const uint4 dq = *(const uint4*)(dY + (((size_t)b * OH + oh) * OW + ow) * C + c8 * 8);
      const __nv_bfloat162* d2 = (const __nv_bfloat162*)&dq;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const float2 f = __bfloat1622float2(d2[k]);
        if (bpos[2 * k] == mine) g[2 * k] += f.x;
        if (bpos[2 * k + 1] == mine) g[2 * k + 1] += f.y;
      }
    }
  __nv_bfloat162 o[4];
#pragma unroll
  for (int k = 0; k < 4; k++) o[k] = __floats2bfloat162_rn(g[2 * k], g[2 * k + 1]);
  *(uint4*)(dX + i * 8) = *(const uint4*)o;
}
// UpsamplingBilinear2d(scale 2, align_corners=True) backward in gather form: input pixel (ih, iw) collects w * dY from the output pixels
// whose 2x2 footprint contains it.  dY [B,2H,2W,C] bf16 -> dX [B,H,W,C] bf16
__global__ void k_upsample_bwd(const bf16* __restrict__ dY, bf16* __restrict__ dX, int B, int H, int W, int C) {
  const int OH = 2 * H, OW = 2 * W;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)B * H * W * C;
  if (i >= n) return;
  const int c = (int)(i % C), iw = (int)((i / C) % W), ih = (int)((i / ((size_t)C * W)) % H), b = (int)(i / ((size_t)C * W * H));
  const float ry = (float)(H - 1) / (float)(OH - 1), rx = (float)(W - 1) / (float)(OW - 1);
  // output rows whose source coordinate fy = oy * ry lies in (ih - 1, ih + 1): oy in (ih-1)/ry .. (ih+1)/ry
  const int oy_lo = max(0, (int)floorf((ih - 1) / ry)), oy_hi = min(OH - 1, (int)ceilf((ih + 1) / ry));
  const int ox_lo = max(0, (int)floorf((iw - 1) / rx)), ox_hi = min(OW - 1, (int)ceilf((iw + 1) / rx));
  float g = 0.f;
  for (int oy = oy_lo; oy <= oy_hi; oy++) {
    const float fy = oy * ry;
    const int y0 = (int)fy, y1 = min(y0 + 1, H - 1);
    const float wy = fy - y0;
    float cy = 0.f;
    if (y0 == ih) cy += 1.f - wy;
    if (y1 == ih) cy += wy;
    if (cy == 0.f) continue;
    for (int ox = ox_lo; ox <= ox_hi; ox++) {
      const float fx = ox * rx;
      const int x0 = (int)fx, x1 = min(x0 + 1, W - 1);
      const float wx = fx - x0;
      float cx = 0.f;
      if (x0 == iw) cx += 1.f - wx;
      if (x1 == iw) cx += wx;
      if (cx == 0.f) continue;
      g += cy * cx * __bfloat162float(dY[(((size_t)b * OH + oy) * OW + ox) * C + c]);
    }
  }
  dX[i] = __float2bfloat16(g);
}
// out = bf16(a + b) (b may be null): sum of the gradients of two branches / fp32 dgrad output -> bf16 activation gradient
__global__ void k_add_to_bf16(const float* __restrict__ a, const float* __restrict__ b, bf16* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = __float2bfloat16(a[i] + (b ? b[i] : 0.f));
}
// out = bf16(a + float(c)) with c bf16 (adds a bf16 gradient branch to an fp32 one)
__global__ void k_add_bf16_to_bf16(const float* __restrict__ a, const bf16* __restrict__ c, bf16* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = __float2bfloat16(a[i] + __bfloat162float(c[i]));
}

// ------------------------------------------------------------------------------------------------ Adam (torch.optim.Adam, weight_decay = L2 added to the gradient)
// p, g, m, v fp32 [n];  step t (1-based):  g' = g + wd p;  m = b1 m + (1-b1) g';  v = b2 v + (1-b2) g'^2;
// p -= lr * (m / (1 - b1^t)) / (sqrt(v / (1 - b2^t)) + eps)          (Grasping_Agent_multidiscrete.py:153-156: lr, wd = 2e-5, defaults otherwise)
__global__ void k_adam(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, size_t n, float lr, float b1, float b2,
                       float eps, float wd, float bc1, float bc2) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gg = g[i] + wd * p[i];
  const float mm = b1 * m[i] + (1.f - b1) * gg, vv = b2 * v[i] + (1.f - b2) * gg * gg;
  m[i] = mm; v[i] = vv;
  p[i] -= lr * (mm / bc1) / (sqrtf(vv / bc2) + eps);
}

// ------------------------------------------------------------------------------------------------ SGD (torch.optim.SGD, dampening 0, nesterov off)
// p, g, buf fp32 [n]:  d = g + wd p;  buf = d (first step) or momentum buf + d;  p -= lr buf        (Grasping_Agent_multidiscrete.py:145-152:
// lr, momentum 0.9, wd 2e-5).  momentum = 0: no buffer, p -= lr d.  Every product and sum is rounded on its own (__fmul_rn / __fadd_rn: no
// contraction into an FMA), in torch's order - mul_(momentum) then add_(d); add_(buf, alpha=-lr).  Where torch's own kernels fuse
// `a + alpha b` into one FMA, the result differs from it by at most half an ulp of wd p and of lr buf.
__global__ void k_sgd(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, size_t n, float lr, float momentum, float wd, int first) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float pp = p[i];
  float d = __fadd_rn(g[i], __fmul_rn(wd, pp));
  if (buf) {
    d = first ? d : __fadd_rn(__fmul_rn(momentum, buf[i]), d);
    buf[i] = d;
  }
  p[i] = __fsub_rn(pp, __fmul_rn(lr, d));
}

// ------------------------------------------------------------------------------------------------ gradient accumulation over micro-batches
// acc = g (first micro-batch) or acc + g, fp32 [n]: torch's .grad accumulation of successive backward() calls, micro-batch 1 first
__global__ void k_grad_accumulate(float* __restrict__ acc, const float* __restrict__ g, size_t n, int first) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  acc[i] = first ? g[i] : __fadd_rn(acc[i], g[i]);
}

// ------------------------------------------------------------------------------------------------ C-ABI
extern "C" int gq_bn_batch_merge(float* stats, int B, int C, void* stream) {
  if (!stats || B <= 0 || C <= 0) { snprintf(q_err, sizeof q_err, "gq_bn_batch_merge: bad argument"); return -1; }
  k_bn_batch_merge<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(stats, B, C);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_bn_running_update(const float* merged_stats, float* running_mean, float* running_var, int B, int HW, int C, float momentum, void* stream) {
  if (!merged_stats || !running_mean || !running_var || B <= 0 || HW <= 0 || C <= 0 || (long long)B * HW < 2) {
    snprintf(q_err, sizeof q_err, "gq_bn_running_update: bad argument");
    return -1;
  }
  k_bn_running_update<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(merged_stats, running_mean, running_var, C, (double)HW, (double)B * HW, (double)momentum);
  QCK(cudaGetLastError());
  return 0;
}
static int loss_head_bwd(const char* what, const float* q, const void* x, const float* w_head, const long long* action, const float* reward, const float* weight,
                         int B, int A, int H, int W, float* loss_terms, float* qsel, void* dX, float* dW_partial, float* db_partial, float* dW_head, float* db_head,
                         void* stream) {
  if (!q || !x || !w_head || !action || !reward || !loss_terms || !qsel || !dX || !dW_partial || !db_partial || !dW_head || !db_head || A > 64) {
    snprintf(q_err, sizeof q_err, "%s: bad argument", what);
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  QCK(cudaMemsetAsync(dX, 0, (size_t)B * H * W * 64 * sizeof(bf16), st));
  k_loss_head_bwd<<<B, 64, 0, st>>>(q, (const bf16*)x, w_head, action, reward, weight, B, A, H, W, loss_terms, qsel, (bf16*)dX, dW_partial, db_partial);
  k_reduce_rows<<<(A * 64 + 127) / 128, 128, 0, st>>>(dW_partial, dW_head, B, (size_t)A * 64);
  k_reduce_rows<<<1, 128, 0, st>>>(db_partial, db_head, B, (size_t)A);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_loss_head_bwd(const float* q, const void* x, const float* w_head, const long long* action, const float* reward, int B, int A, int H, int W,
                                float* loss_terms, float* qsel, void* dX, float* dW_partial, float* db_partial, float* dW_head, float* db_head, void* stream) {
  return loss_head_bwd("gq_loss_head_bwd", q, x, w_head, action, reward, nullptr, B, A, H, W, loss_terms, qsel, dX, dW_partial, db_partial, dW_head, db_head, stream);
}
extern "C" int gq_loss_head_bwd_weighted(const float* q, const void* x, const float* w_head, const long long* action, const float* reward, const float* weight,
                                         int B, int A, int H, int W, float* loss_terms, float* qsel, void* dX, float* dW_partial, float* db_partial, float* dW_head,
                                         float* db_head, void* stream) {
  if (!weight) { snprintf(q_err, sizeof q_err, "gq_loss_head_bwd_weighted: bad argument"); return -1; }
  return loss_head_bwd("gq_loss_head_bwd_weighted", q, x, w_head, action, reward, weight, B, A, H, W, loss_terms, qsel, dX, dW_partial, db_partial, dW_head,
                       db_head, stream);
}
extern "C" int gq_bn_relu_bwd(const void* dY, const void* act, const float* o, const float* stats, const float* gamma, int B, int HW, int C, float eps,
                              void* dpre_out, float* scratch_part, float* scratch_sums, float* dgamma, float* dbeta, void* d_o, void* stream) {
  if (!dY || !act || !o || !stats || !gamma || !scratch_part || !scratch_sums || !d_o) { snprintf(q_err, sizeof q_err, "gq_bn_relu_bwd: bad argument"); return -1; }
  if (C % 8) { snprintf(q_err, sizeof q_err, "gq_bn_relu_bwd: C must be a multiple of 8"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  const int rows = B * HW, rpc = 128, nparts = (rows + rpc - 1) / rpc;
  k_bn_bwd_reduce<<<nparts, 256, 0, st>>>((const bf16*)dY, (const bf16*)act, o, stats, rows, C, HW, eps, rpc, (bf16*)dpre_out, scratch_part);
  k_bn_bwd_sums<<<(C + 3) / 4, 128, 0, st>>>(scratch_part, nparts, C, scratch_sums, dgamma, dbeta);
  const size_t n = (size_t)rows * C;
  k_bn_bwd_apply8<<<(unsigned)((n / 8 + 255) / 256), 256, 0, st>>>((const bf16*)dY, (const bf16*)act, o, stats, gamma, scratch_sums, n / 8, C, HW, 1.f / (float)rows, eps,
                                                                     (bf16*)d_o);
  QCK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------ weight gradient on wgmma
// dW[co][tap][ci] = sum over images b and pixels p of dY[b,p,co] * X[b, p + tap, ci]  (zero outside the image), as a tensor-core GEMM:
// D[co][ci] (one filter tap, one image) = sum over pixels p of dY[p][co] * X[p + tap][ci],
// i.e. M = 128 output channels, N = BLOCK_N input channels, K = pixels.  Both operands are pixel-major in memory ([pixel][channel], NHWC), so
// with K = pixels they are **MN-major** wgmma operands: a shared-memory tile is K rows (pixels) of 128 bytes (64 channels), 8 rows = one
// 1024-byte swizzle atom - exactly the image a 128-byte-swizzled TMA box of [64 channels x 128 pixels] leaves.  Canonical MN-major
// SWIZZLE_128B layout: the next 64 channels (second box) LBO = 16 384 bytes further, the next 8 pixels SBO = 1024 bytes further; one
// wgmma (K = 16) consumes 16 rows = 2048 bytes.
//   A = dY: 3-D tiled map [Cout][H*W][B], box 64 x 128 x 1 - rows past the end of the image are out of bounds and read as zeros, so the
//           last k-step of an image contributes nothing for them whatever the X load returns there;
//   B = X : the forward's im2col-mode map (tap passed as offsets, zero fill = convolution padding): 128 consecutive output positions.
// grid (ceil(Cout / 128), Cin / BLOCK_N, taps * B); split-K over the images (partials [B][Cout][taps][Cin], summed in image
// order by k_reduce_rows: deterministic).  Roles as in k_conv_wgmma: warp 8 lane 0 TMA producer, warpgroup g = 0, 1 multiplies and stores
// output channels co0 + 64 g .. co0 + 64 g + 63 (its own dY box).
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem_addr, const CUtensorMap* tmap, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(dst_smem_addr), "l"((uint64_t)tmap), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
#define WT_K 128                      // pixels per k-step (= the im2col map's pixels per column)
#define WT_BOX (WT_K * 128)           // bytes of one [64 channels x 128 pixels] box
template <int BLOCK_N, int STAGES>
__global__ void __launch_bounds__(CONV_THREADS, 1) k_wgrad_wgmma(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                                                                float* __restrict__ part, int H, int W, int Cin, int Cout, int ks) {
  constexpr int A_STAGE = 2 * WT_BOX, B_STAGE = (BLOCK_N / 64) * WT_BOX;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_STAGE;
  uint64_t* full = (uint64_t*)(smem + STAGES * (A_STAGE + B_STAGE));
  uint64_t* empty = full + STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int taps = ks * ks, pad = ks / 2, HW = H * W, nk = (HW + WT_K - 1) / WT_K;
  const int co0 = blockIdx.x * 128, ci0 = blockIdx.y * BLOCK_N, tap = blockIdx.z % taps, b = blockIdx.z / taps;
  if (tid == 0) {
    for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  if (warp == 8) {
    if (lane == 0) {
      for (int kn = 0; kn < nk; kn++) {
        const int s = kn % STAGES, round = kn / STAGES;
        if (round > 0) mbar_wait(&empty[s], (uint32_t)(round - 1) & 1u);
        mbar_arrive_expect_tx(&full[s], (uint32_t)(A_STAGE + B_STAGE));
        const int p0 = kn * WT_K, oh0 = p0 / W, ow0 = p0 - oh0 * W;
        const uint32_t a_dst = smem_u32(sA) + (uint32_t)(s * A_STAGE), b_dst = smem_u32(sB) + (uint32_t)(s * B_STAGE);
        tma_load_3d(a_dst, &tmap_dy, co0, p0, b, &full[s]);
        tma_load_3d(a_dst + WT_BOX, &tmap_dy, co0 + 64, p0, b, &full[s]);  // (Cout = 64: wholly out of bounds -> zeros, rows 64..127 of D unused)
#pragma unroll
        for (int j = 0; j < BLOCK_N / 64; j++)
          tma_load_im2col_4d(b_dst + (uint32_t)(j * WT_BOX), &tmap_x, ci0 + j * 64, ow0 - pad, oh0 - pad, b, (uint16_t)(tap % ks), (uint16_t)(tap / ks), &full[s]);
      }
    }
    return;
  }
  const int wg = warp >> 2;
  float acc[BLOCK_N / 2];
#pragma unroll
  for (int i = 0; i < BLOCK_N / 2; i++) acc[i] = 0.f;
  int s = 0, prev = -1;
  uint32_t ph = 0;
  for (int kb = 0; kb < nk; kb++) {
    mbar_wait(&full[s], ph);
    const uint32_t a_base = smem_u32(sA + s * A_STAGE) + (uint32_t)(wg * WT_BOX), b_base = smem_u32(sB + s * B_STAGE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < WT_K / 16; k++)
      wgmma_tile<BLOCK_N, 1, 1>(acc, gmma_desc_sw128(a_base + k * 2048, WT_BOX), gmma_desc_sw128(b_base + k * 2048, WT_BOX), (kb > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1u; }
  }
  wgmma_wait<0>();
  // fragment: output channel co0 + 64 wg + 16 (warp % 4) + lane / 4 (+ 8), input channels ci0 + 8 j + 2 (lane % 4) + {0, 1}
  const int coa = co0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), cob = coa + 8;
  float* rowa = part + (((size_t)b * Cout + (coa < Cout ? coa : 0)) * taps + tap) * Cin + ci0;
  float* rowb = part + (((size_t)b * Cout + (cob < Cout ? cob : 0)) * taps + tap) * Cin + ci0;
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; j++) {
    const int c = 8 * j + 2 * (lane & 3);
    if (coa < Cout) *(float2*)(rowa + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
    if (cob < Cout) *(float2*)(rowb + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// 3-D tiled tensor map of dY [B][H*W][Cout] bf16 (innermost first: Cout, H*W, B) with a [64 channels x 128 pixels x 1 image] box
typedef CUresult (*EncodeTiledFn3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int make_dy_tmap(CUtensorMap* m, const void* dy, int B, int HW, int Cout) {
  static EncodeTiledFn3 fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn3)p;
  }
  if (!fn) { snprintf(q_err, sizeof q_err, "cuTensorMapEncodeTiled is not available"); return -3; }
  cuuint64_t gdim[3] = {(cuuint64_t)Cout, (cuuint64_t)HW, (cuuint64_t)B};
  cuuint64_t gstride[2] = {(cuuint64_t)Cout * 2, (cuuint64_t)HW * Cout * 2};
  cuuint32_t box[3] = {64, WT_K, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(dy), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(q_err, sizeof q_err, "cuTensorMapEncodeTiled (dY) failed (%d)", (int)r); return -3; }
  return 0;
}
// -> 0 launched, < 0 error (q_err set)
static int launch_wgrad_tc(cudaStream_t st, const void* dY, const void* x, float* part, int B, int H, int W, int Cin, int Cout, int ks) {
  alignas(64) CUtensorMap tdy, tx;
  memset(&tdy, 0, sizeof tdy); memset(&tx, 0, sizeof tx);
  int r = make_dy_tmap(&tdy, dY, B, H * W, Cout);
  if (r == 0) r = make_act_tmap_im2col(&tx, x, B, H, W, Cin, ks);
  if (r) return r;
  const int taps = ks * ks;
#define LAUNCH_WT(BN_, ST_)                                                                                                   \
  do {                                                                                                                        \
    const size_t smem = 1024 + (size_t)ST_ * (2 * WT_BOX + (BN_ / 64) * WT_BOX) + 16 * ST_;                                    \
    QCK(cudaFuncSetAttribute(k_wgrad_wgmma<BN_, ST_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                \
    dim3 grid((Cout + 127) / 128, Cin / BN_, taps * B);                                                                       \
    k_wgrad_wgmma<BN_, ST_><<<grid, CONV_THREADS, smem, st>>>(tdy, tx, part, H, W, Cin, Cout, ks);                             \
  } while (0)
  if (Cin % 128 == 0) LAUNCH_WT(128, 3);
  else LAUNCH_WT(64, 4);
#undef LAUNCH_WT
  return 0;
}

// scratch_part of gq_bn_relu_bwd: ceil(B*HW / 128) * C * 2 floats
extern "C" int gq_conv_wgrad(const void* dY, const void* x, float* scratch_part, float* dW, int B, int H, int W, int Cin, int Cout, int ks, void* stream) {
  if (!dY || !x || !scratch_part || !dW || (ks != 1 && ks != 3) || Cin % 64 || Cout % 64) { snprintf(q_err, sizeof q_err, "gq_conv_wgrad: bad argument"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  const int taps = ks * ks;
  const int r = launch_wgrad_tc(st, dY, x, scratch_part, B, H, W, Cin, Cout, ks);
  if (r) return r;
  const size_t n = (size_t)Cout * taps * Cin;
  k_reduce_rows<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(scratch_part, dW, B, n);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_conv_first_wgrad(const void* dY, const float* x, float* scratch_part, float* dW, int B, int H, int W, void* stream) {
  if (!dY || !x || !scratch_part || !dW || (long long)B * H * W >= (1LL << 31)) { snprintf(q_err, sizeof q_err, "gq_conv_first_wgrad: bad argument"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)B * H * W;
  const int ppc = 2048, chunks = (int)((n + ppc - 1) / ppc);
  k_conv_first_wgrad<<<chunks, 256, 0, st>>>((const bf16*)dY, x, scratch_part, B, H, W, ppc);
  k_reduce_rows<<<(64 * 36 + 127) / 128, 128, 0, st>>>(scratch_part, dW, chunks, (size_t)64 * 36);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_maxpool_bwd(const void* x, const void* dY, void* dX, int B, int H, int W, int C, void* stream) {
  if (C % 8) { snprintf(q_err, sizeof q_err, "gq_maxpool_bwd: C must be a multiple of 8"); return -1; }
  const size_t n = (size_t)B * H * W * C;
  k_maxpool_bwd8<<<(unsigned)((n / 8 + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)dY, (bf16*)dX, B, H, W, C);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_upsample2x_bwd(const void* dY, void* dX, int B, int H, int W, int C, void* stream) {
  const size_t n = (size_t)B * H * W * C;
  k_upsample_bwd<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)dY, (bf16*)dX, B, H, W, C);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_add_to_bf16(const float* a, const float* b, const void* c_bf16, void* out, size_t n, void* stream) {
  if (!a || !out || (b && c_bf16)) { snprintf(q_err, sizeof q_err, "gq_add_to_bf16: bad argument"); return -1; }
  if (c_bf16) k_add_bf16_to_bf16<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, (const bf16*)c_bf16, (bf16*)out, n);
  else k_add_to_bf16<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, b, (bf16*)out, n);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_adam(float* p, const float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                       void* stream) {
  if (!p || !g || !m || !v || step < 1) { snprintf(q_err, sizeof q_err, "gq_adam: bad argument"); return -1; }
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  k_adam<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_sgd(float* p, const float* g, float* buf, size_t n, float lr, float momentum, float weight_decay, int first, void* stream) {
  if (!p || !g || (momentum != 0.f && !buf) || !(momentum >= 0.f)) { snprintf(q_err, sizeof q_err, "gq_sgd: bad argument"); return -1; }
  if (n == 0) return 0;
  k_sgd<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, g, momentum != 0.f ? buf : nullptr, n, lr, momentum, weight_decay, first);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_grad_accumulate(float* acc, const float* g, size_t n, int first, void* stream) {
  if (!acc || !g) { snprintf(q_err, sizeof q_err, "gq_grad_accumulate: bad argument"); return -1; }
  if (n == 0) return 0;
  k_grad_accumulate<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(acc, g, n, first);
  QCK(cudaGetLastError());
  return 0;
}
