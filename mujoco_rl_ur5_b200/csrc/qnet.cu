// libgrasp_qnet.so — forward pass of the pixel-wise grasp Q-network (reference: Modules.py:308-311 MULTIDISCRETE_RESNET =
// Perception_Module :159-193 + Grasping_Module_multidiscrete :243-287, BasicBlock :92-142) over a batch of environments.
//
// bf16 activations (NHWC) and weights, fp32 accumulation.  The 3x3 / 1x1 convolutions with Cin >= 64 (>99.9 % of the MACs) run
// as implicit GEMMs on the Hopper tensor cores: both operands are brought into 128-byte-swizzled K-major shared-memory tiles by TMA
// (an im2col-mode map for the activations, a tiled map for the weights), completion tracked with mbarrier transaction counts, and
// two consumer warpgroups multiply them with wgmma.mma_async (m64 x N x k16, accumulator in registers).  BatchNorm uses per-image
// batch statistics because the reference never puts the policy net in eval() and forwards one image at a time (SURVEY 3.4, quirk Q9).
//
// C-ABI: see include/grasp_qnet.h.  No CPU fallback.
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched with cudaGetDriverEntryPoint, libcuda is not linked)
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/grasp_qnet.h"

typedef __nv_bfloat16 bf16;

static thread_local char q_err[256] = "";
extern "C" const char* gq_last_error(void) { return q_err; }
#define QCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { snprintf(q_err, sizeof q_err, "CUDA error: %s", cudaGetErrorString(e_)); return -2; } } while (0)

// ------------------------------------------------------------------------------------------------ small PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0, addr = smem_u32(bar);
  while (!done) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(addr), "r"(parity) : "memory");
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// TMA: one thread copies a whole box into a 128-byte-swizzled shared-memory tile; completion is reported to the mbarrier as
// transferred bytes (complete_tx)
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem_addr, const CUtensorMap* tmap, int x, int y, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst_smem_addr), "l"((uint64_t)tmap), "r"(x), "r"(y), "r"(smem_u32(bar)) : "memory");
}
// im2col mode: the 128 consecutive output positions starting at pixel (w, h) of image n, for filter tap (off_w, off_h), 64 channels from c;
// hardware zero fill outside the image (the convolution padding)
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst_smem_addr, const CUtensorMap* tmap, int c, int w, int h, int n, uint16_t off_w,
                                                   uint16_t off_h, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
               ::"r"(dst_smem_addr), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h) : "memory");
}

// ---- wgmma (sm_90a).  A and B both from shared memory; TA / TB = 1 marks an MN-major operand (the weight gradient), 0 a K-major one.
// Shared-memory matrix descriptor, SWIZZLE_128B: start address, leading byte offset (MN-major: distance of the next 64-element block
// along M / N; unused for K-major), stride byte offset (distance of the next 8-row group: 8 x 128 B), layout type 1 = 128-byte swizzle.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}
// D (+)= A * B for one warpgroup: 64 rows x BLOCK_N columns, K = 16
template <int BLOCK_N, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&d)[BLOCK_N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (BLOCK_N == 128) wgmma_m64n128<TA, TB>(d, adesc, bdesc, accumulate);
  else wgmma_m64n64<TA, TB>(d, adesc, bdesc, accumulate);
}

// ------------------------------------------------------------------------------------------------ implicit-GEMM convolution on wgmma
// x  [B,H,W,Cin] bf16 (NHWC), w [Cout][ks*ks][Cin] bf16, y [B,H,W,Cout] f32 (+ bias), partials [B][gx][8][Cout][2] f32 (sum, sum of squares)
// One tile = 128 output pixels (BM) x BLOCK_N output channels of one image, walked in k-steps of 64 input channels of one filter tap.
// Persistent: CTA i takes tiles i, i + gridDim.x, ... (m tile fastest, then n tile, then image).  288 threads: warpgroups 0 and 1
// consume (rows 0-63 / 64-127 of the tile), warp 8 lane 0 produces.  One k-step = one arrive.expect_tx(A + B bytes) on the stage's
// full barrier (count 1) and two TMAs: the im2col box of the activations (128 output positions x 64 channels for the tap, zero fill
// at the image border) and the [BLOCK_N x 64] box of the weights, both 128-byte swizzled K-major.  A consumer warpgroup issues the
// four k16 wgmmas of a stage, keeps one group in flight and releases the previous stage (empty barrier, one arrival per consumer warp,
// count 8) once wgmma.wait_group 1 says its reads are done.  The producer runs ahead across tile boundaries, so the loads of the next
// tile overlap the epilogue of the current one.
#define BM 128
#define BK 64
#define CONV_THREADS 288
#define CONV_PARTS 8  // BatchNorm partial rows per tile: one per consumer warp (gq_conv_partials_floats)
// epilogue of one warpgroup's 64 x BLOCK_N accumulator (wgmma fragment: row 16 warp + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) + {0, 1})
//   EPI 0: y = conv + bias (fp32) and, if requested, per-(tile, warp) BatchNorm partials over the warp's 16 rows, reduced over the
//          lanes in a fixed order (deterministic) and summed in a fixed order by k_bn_reduce
//   EPI 1 (BasicBlock tail): out = relu(resid * scale + shift + conv + bias) as bf16 (BasicBlock.forward, Modules.py:128-142)
//   EPI 2 (BatchNorm folded into the weights, eval mode): out = conv + bias as bf16, ReLU if `relu`
template <int BLOCK_N, int EPI>
__device__ __forceinline__ void conv_epilogue(const float (&acc)[BLOCK_N / 2], int wg, int warp, int lane, int mt, int n0, int b, int gx, int HW, int Cout,
                                              const float* __restrict__ bias, float* __restrict__ y, float* __restrict__ stats,
                                              const float* __restrict__ resid, const float2* __restrict__ scale_shift, bf16* __restrict__ out, int relu) {
  const int wq = warp & 3;
  const int ma = mt * BM + wg * 64 + wq * 16 + (lane >> 2), mb = ma + 8;
  const bool va = ma < HW, vb = mb < HW;
  const size_t rowa = ((size_t)b * HW + ma) * Cout, rowb = ((size_t)b * HW + mb) * Cout;
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; j++) {
    const int c = n0 + 8 * j + 2 * (lane & 3);
    float x0 = acc[4 * j], x1 = acc[4 * j + 1], x2 = acc[4 * j + 2], x3 = acc[4 * j + 3];
    if (bias) { const float2 bv = __ldg((const float2*)(bias + c)); x0 += bv.x; x1 += bv.y; x2 += bv.x; x3 += bv.y; }
    if constexpr (EPI == 0) {
      if (va) *(float2*)(y + rowa + c) = make_float2(x0, x1);
      if (vb) *(float2*)(y + rowb + c) = make_float2(x2, x3);
      if (stats) {
        if (!va) { x0 = 0.f; x1 = 0.f; }
        if (!vb) { x2 = 0.f; x3 = 0.f; }
        float s0 = x0 + x2, s1 = x1 + x3, q0 = x0 * x0 + x2 * x2, q1 = x1 * x1 + x3 * x3;
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          q0 += __shfl_xor_sync(0xffffffffu, q0, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
        }
        if (lane < 4) *(float4*)(stats + ((((size_t)b * gx + mt) * CONV_PARTS + wg * 4 + wq) * Cout + c) * 2) = make_float4(s0, q0, s1, q1);
      }
    } else if constexpr (EPI == 2) {
      if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); x2 = fmaxf(x2, 0.f); x3 = fmaxf(x3, 0.f); }
      if (va) *(__nv_bfloat162*)(out + rowa + c) = __floats2bfloat162_rn(x0, x1);
      if (vb) *(__nv_bfloat162*)(out + rowb + c) = __floats2bfloat162_rn(x2, x3);
    } else {
      const float4 ss = __ldg((const float4*)(scale_shift + (size_t)b * Cout + c));  // (scale, shift) of columns c, c + 1
      if (va) {
        const float2 r = __ldg((const float2*)(resid + rowa + c));
        *(__nv_bfloat162*)(out + rowa + c) = __floats2bfloat162_rn(fmaxf(r.x * ss.x + ss.y + x0, 0.f), fmaxf(r.y * ss.z + ss.w + x1, 0.f));
      }
      if (vb) {
        const float2 r = __ldg((const float2*)(resid + rowb + c));
        *(__nv_bfloat162*)(out + rowb + c) = __floats2bfloat162_rn(fmaxf(r.x * ss.x + ss.y + x2, 0.f), fmaxf(r.y * ss.z + ss.w + x3, 0.f));
      }
    }
  }
}
// Optional second A source (Cx > 0): after the ks*ks taps x Cin/64 chunks of the convolution of x, the K loop runs on over Cx/64 chunks
// of a 1x1 convolution of x2 (its own im2col map), accumulating into the same registers; the weights are one [Cout][ks*ks*Cin + Cx]
// matrix, so only the producer's choice of activation map and coordinates depends on the source.
template <int BLOCK_N, int STAGES, int EPI>
__global__ void __launch_bounds__(CONV_THREADS, 1) k_conv_wgmma(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                                                               const __grid_constant__ CUtensorMap tmap_x2, const float* __restrict__ bias,
                                                               float* __restrict__ y, float* __restrict__ stats, const float* __restrict__ resid,
                                                               const float2* __restrict__ scale_shift, bf16* __restrict__ out, int H, int W, int Cin, int Cx,
                                                               int Cout, int ks, int relu, int gx, int gy, int ntiles) {
  constexpr int A_STAGE = BM * BK * 2, B_STAGE = BLOCK_N * BK * 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);  // the 128-byte swizzle pattern repeats every 1024 bytes
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_STAGE;
  uint64_t* full = (uint64_t*)(smem + STAGES * (A_STAGE + B_STAGE));
  uint64_t* empty = full + STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int HW = H * W, pad = ks / 2, kchunks = Cin / BK, nk_a = ks * ks * kchunks, nk = nk_a + Cx / BK;
  if (tid == 0) {
    for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  if (warp == 8) {
    if (lane == 0) {
      int sn = 0, round = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int mt = t % gx, nt = (t / gx) % gy, b = t / (gx * gy);
        const int m0 = mt * BM, n0 = nt * BLOCK_N;
        const int oh0 = m0 / W, ow0 = m0 - oh0 * W;
        int tap = 0, kc = 0;
        for (int kn = 0; kn < nk; kn++) {
          if (round > 0) mbar_wait(&empty[sn], (uint32_t)(round - 1) & 1u);
          mbar_arrive_expect_tx(&full[sn], (uint32_t)(A_STAGE + B_STAGE));
          if (kn < nk_a) {
            tma_load_im2col_4d(smem_u32(sA) + (uint32_t)(sn * A_STAGE), &tmap_x, kc * BK, ow0 - pad, oh0 - pad, b, (uint16_t)(tap % ks), (uint16_t)(tap / ks),
                               &full[sn]);
            if (++kc == kchunks) { kc = 0; tap++; }
          } else {
            tma_load_im2col_4d(smem_u32(sA) + (uint32_t)(sn * A_STAGE), &tmap_x2, (kn - nk_a) * BK, ow0, oh0, b, 0, 0, &full[sn]);
          }
          tma_load_2d(smem_u32(sB) + (uint32_t)(sn * B_STAGE), &tmap_w, kn * BK, n0, &full[sn]);
          if (++sn == STAGES) { sn = 0; round++; }
        }
      }
    }
    return;
  }
  const int wg = warp >> 2;
  int s = 0;
  uint32_t ph = 0;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int mt = t % gx, nt = (t / gx) % gy, b = t / (gx * gy);
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i++) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < nk; kb++) {
      mbar_wait(&full[s], ph);
      const uint32_t a_base = smem_u32(sA + s * A_STAGE) + (uint32_t)(wg * 64 * 128), b_base = smem_u32(sB + s * B_STAGE);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; k++)  // K = 16 bf16 = 32 bytes further inside the swizzle atom
        wgmma_tile<BLOCK_N, 0, 0>(acc, gmma_desc_sw128(a_base + k * 32, 16), gmma_desc_sw128(b_base + k * 32, 16), (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();  // the wgmmas of the previous stage have completed: release it
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);
    conv_epilogue<BLOCK_N, EPI>(acc, wg, warp, lane, mt, nt * BLOCK_N, b, gx, HW, Cout, bias, y, stats, resid, scale_shift, out, relu);
  }
}

// per-image BatchNorm (training mode, own statistics) folded into one multiply-add per channel: (scale, shift) from (sum, sum of squares)
__global__ void k_bn_scale_shift(const float* __restrict__ stats, const float* __restrict__ gamma, const float* __restrict__ beta, float2* __restrict__ ss,
                                 int B, int C, int HW, float eps) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  int c = i % C;
  float s1 = stats[(size_t)i * 2], s2 = stats[(size_t)i * 2 + 1];
  float mean = s1 / HW, var = fmaxf(s2 / HW - mean * mean, 0.f);  // same expressions as k_bn_act
  float scale = rsqrtf(var + eps) * gamma[c];
  ss[i] = make_float2(scale, beta[c] - mean * scale);
}

// per-image batch-norm statistics from the per-(tile, warp) partials of k_conv_wgmma, summed in a fixed order (double accumulation)
__global__ void k_bn_reduce(const float* __restrict__ part, float* __restrict__ stats, int B, int nparts, int C) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  int b = i / C, c = i % C;
  // one accumulator pair in part order (the order is part of the result); the unrolled body keeps 8 independent 8-byte loads in flight
  // (a 4-accumulator version with a dynamically indexed remainder goes to local memory)
  double s1 = 0, s2 = 0;
  const float2* p = (const float2*)part + (size_t)b * nparts * C + c;
#pragma unroll 8
  for (int k = 0; k < nparts; k++) { const float2 v = __ldg(p + (size_t)k * C); s1 += v.x; s2 += v.y; }
  stats[(size_t)i * 2] = (float)s1; stats[(size_t)i * 2 + 1] = (float)s2;
}

// ------------------------------------------------------------------------------------------------ small layers
// first conv: x [B,4,H,W] f32 (NCHW, the agent's tensor), w [64][3][3][4] f32 -> y [B,H,W,64] bf16; no BN / ReLU follows (Modules.py:176).
// Two consecutive pixels of the flattened index per thread: every weight vector read from shared memory feeds both (half the LDS
// traffic per FMA of a kernel with one pixel per thread).  When B*H*W is odd, the last thread computes its one pixel twice and stores it once
// (clamping its index keeps 126 registers = four CTAs per SM; selecting the pixel took 130 registers and left room for three).
__global__ void __launch_bounds__(128) k_conv_first2(const float* __restrict__ x, const float* __restrict__ w, bf16* __restrict__ y, int B, int H, int W) {
  __shared__ __align__(16) float sw[64 * 36];
  for (int i = threadIdx.x; i < 64 * 36; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int HW = H * W;
  const int p0 = 2 * (blockIdx.x * blockDim.x + threadIdx.x);
  if (p0 >= B * HW) return;
  float in[2][36];
#pragma unroll
  for (int q = 0; q < 2; q++) {
    const int p = min(p0 + q, B * HW - 1), b = p / HW, oh = (p % HW) / W, ow = p % W;
#pragma unroll
    for (int t = 0; t < 9; t++) {
      const int ih = oh + t / 3 - 1, iw = ow + t % 3 - 1;
      const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
#pragma unroll
      for (int c = 0; c < 4; c++) in[q][t * 4 + c] = ok ? __ldg(x + ((size_t)(b * 4 + c) * H + ih) * W + iw) : 0.f;
    }
  }
  bf16* out = y + (size_t)p0 * 64;
  const float4* sw4 = (const float4*)sw;
  for (int co = 0; co < 64; co += 8) {
    __nv_bfloat162 o[2][4];
#pragma unroll
    for (int h = 0; h < 4; h++) {
      float a[2][2] = {{0, 0}, {0, 0}};
#pragma unroll
      for (int k = 0; k < 9; k++) {
        const float4 w0 = sw4[(co + 2 * h) * 9 + k], w1 = sw4[(co + 2 * h + 1) * 9 + k];
#pragma unroll
        for (int q = 0; q < 2; q++) {  // every output: one chain over the taps and input channels in order, whatever the pixel count
          a[q][0] += in[q][4 * k] * w0.x; a[q][0] += in[q][4 * k + 1] * w0.y; a[q][0] += in[q][4 * k + 2] * w0.z; a[q][0] += in[q][4 * k + 3] * w0.w;
          a[q][1] += in[q][4 * k] * w1.x; a[q][1] += in[q][4 * k + 1] * w1.y; a[q][1] += in[q][4 * k + 2] * w1.z; a[q][1] += in[q][4 * k + 3] * w1.w;
        }
      }
      o[0][h] = __floats2bfloat162_rn(a[0][0], a[0][1]); o[1][h] = __floats2bfloat162_rn(a[1][0], a[1][1]);
    }
    *(uint4*)(out + co) = *(uint4*)o[0];
    if (p0 + 1 < B * HW) *(uint4*)(out + 64 + co) = *(uint4*)o[1];
  }
}
// MaxPool2d(kernel 3, stride 2, padding 1) on NHWC bf16
__global__ void k_maxpool(const bf16* __restrict__ x, bf16* __restrict__ y, int B, int H, int W, int C) {
  int OH = (H + 1) / 2, OW = (W + 1) / 2, vc = C / 8;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)B * OH * OW * vc;
  if (i >= n) return;
  int cv = (i % vc) * 8;
  size_t p = i / vc;
  int ow = p % OW, oh = (p / OW) % OH, b = p / ((size_t)OW * OH);
  float m[8];
#pragma unroll
  for (int k = 0; k < 8; k++) m[k] = -3.0e38f;
  for (int dh = -1; dh <= 1; dh++) for (int dw = -1; dw <= 1; dw++) {
    int ih = 2 * oh + dh, iw = 2 * ow + dw;
    if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
    uint4 qv = __ldg((const uint4*)(x + (((size_t)b * H + ih) * W + iw) * C + cv));
    const __nv_bfloat162* pv = (const __nv_bfloat162*)&qv;
#pragma unroll
    for (int k = 0; k < 4; k++) { float2 v = __bfloat1622float2(pv[k]); m[2 * k] = fmaxf(m[2 * k], v.x); m[2 * k + 1] = fmaxf(m[2 * k + 1], v.y); }
  }
  __nv_bfloat162 o[4];
#pragma unroll
  for (int k = 0; k < 4; k++) o[k] = __floats2bfloat162_rn(m[2 * k], m[2 * k + 1]);
  *(uint4*)(y + p * C + cv) = *(uint4*)o;
}
// y = relu( (x - mean) * rstd * gamma + beta [+ identity] ), per-image statistics from `stats` (sum, sumsq over H*W); fp32 in, bf16 out
// one CTA = a run of pixels of one image: per-channel scale / shift (training-mode BatchNorm with the image's own statistics) are
// prepared once in shared memory, then every thread streams 8 channels at a time (2 x 16 B in, 16 B out)
__global__ void __launch_bounds__(256) k_bn_act(const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                                                const float* __restrict__ beta, const float* __restrict__ identity, bf16* __restrict__ y, int HW, int C,
                                                float eps, int pix_per_cta) {
  extern __shared__ float sc[];  // scale[C], shift[C]
  const int b = blockIdx.y, tid = threadIdx.x;
  for (int c = tid; c < C; c += blockDim.x) {
    float s1 = stats[((size_t)b * C + c) * 2], s2 = stats[((size_t)b * C + c) * 2 + 1];
    float mean = s1 / HW, var = fmaxf(s2 / HW - mean * mean, 0.f);  // biased variance, as BatchNorm uses for normalisation
    float scale = rsqrtf(var + eps) * gamma[c];
    sc[c] = scale; sc[C + c] = beta[c] - mean * scale;
  }
  __syncthreads();
  const int vc = C / 8, p0 = blockIdx.x * pix_per_cta, np = min(HW, p0 + pix_per_cta) - p0;
  const size_t base = ((size_t)b * HW + p0) * C;
  for (int i = tid; i < np * vc; i += blockDim.x) {
    const int cv = (i % vc) * 8;
    const size_t off = base + (size_t)(i / vc) * C + cv;
    float v[8];
    *(float4*)v = __ldg((const float4*)(x + off)); *(float4*)(v + 4) = __ldg((const float4*)(x + off + 4));
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = v[k] * sc[cv + k] + sc[C + cv + k];
    if (identity) {
      float r[8];
      *(float4*)r = __ldg((const float4*)(identity + off)); *(float4*)(r + 4) = __ldg((const float4*)(identity + off + 4));
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] += r[k];
    }
    __nv_bfloat162 o[4];
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = __floats2bfloat162_rn(fmaxf(v[2 * k], 0.f), fmaxf(v[2 * k + 1], 0.f));
    *(uint4*)(y + off) = *(uint4*)o;
  }
}
// nn.UpsamplingBilinear2d(scale_factor=2) = bilinear, align_corners=True; NHWC bf16, 8 channels (16 B) per thread
__global__ void k_upsample2x(const bf16* __restrict__ x, bf16* __restrict__ y, int B, int H, int W, int C) {
  int OH = 2 * H, OW = 2 * W, vc = C / 8;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)B * OH * OW * vc;
  if (i >= n) return;
  int cv = (i % vc) * 8;
  size_t p = i / vc;
  int ow = p % OW, oh = (p / OW) % OH, b = p / ((size_t)OW * OH);
  float fy = oh * (float)(H - 1) / (float)(OH - 1), fx = ow * (float)(W - 1) / (float)(OW - 1);
  int y0 = (int)fy, x0 = (int)fx, y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  float wy = fy - y0, wx = fx - x0;
  auto at = [&](int yy, int xx) { return __ldg((const uint4*)(x + (((size_t)b * H + yy) * W + xx) * C + cv)); };
  uint4 qa = at(y0, x0), qb = at(y0, x1), qc = at(y1, x0), qd = at(y1, x1);
  const __nv_bfloat162 *pa = (const __nv_bfloat162*)&qa, *pb = (const __nv_bfloat162*)&qb, *pc = (const __nv_bfloat162*)&qc, *pd = (const __nv_bfloat162*)&qd;
  __nv_bfloat162 o[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    float2 a = __bfloat1622float2(pa[k]), bb = __bfloat1622float2(pb[k]), cc = __bfloat1622float2(pc[k]), d = __bfloat1622float2(pd[k]);
    float r0 = (a.x * (1 - wx) + bb.x * wx) * (1 - wy) + (cc.x * (1 - wx) + d.x * wx) * wy;
    float r1 = (a.y * (1 - wx) + bb.y * wx) * (1 - wy) + (cc.y * (1 - wx) + d.y * wx) * wy;
    o[k] = __floats2bfloat162_rn(r0, r1);
  }
  *(uint4*)(y + p * C + cv) = *(uint4*)o;
}
// The head's arithmetic, shared by gq_head_up2 (k_head + k_up2_sigmoid) and gq_head_max_target (k_head_max): the maximum of the
// target network must be one of the Q-values of the forward, bit for bit, so both paths evaluate the same expressions.
// the pixel's 64 channels (8 x 16 bytes of bf16) as floats
__device__ __forceinline__ void head_load_pixel(const bf16* __restrict__ px, float (&in)[64]) {
  const uint4* src = (const uint4*)px;
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const uint4 qv = __ldg(src + c);
    const __nv_bfloat162* pv = (const __nv_bfloat162*)&qv;
#pragma unroll
    for (int k = 0; k < 4; k++) { float2 v = __bfloat1622float2(pv[k]); in[8 * c + 2 * k] = v.x; in[8 * c + 2 * k + 1] = v.y; }
  }
}
// output plane a of the 1x1 convolution at one pixel; sw = the weights [A][64] f32 in shared memory, the biases at sw[8 * 64 + a]
__device__ __forceinline__ float head_dot(const float (&in)[64], const float* sw, int a) {
  float acc = sw[8 * 64 + a];
#pragma unroll
  for (int c = 0; c < 16; c++) {
    float4 wv = ((const float4*)sw)[a * 16 + c];
    acc += in[4 * c] * wv.x; acc += in[4 * c + 1] * wv.y; acc += in[4 * c + 2] * wv.z; acc += in[4 * c + 3] * wv.w;
  }
  return acc;
}
// source taps of output row (or column) o of UpsamplingBilinear2d(2) (align_corners=True) from n rows: rows i0, i1, weight w of i1
struct Up2Tap { int i0, i1; float w; };
__device__ __forceinline__ Up2Tap up2_tap(int o, int n) {
  const float f = o * (float)(n - 1) / (float)(2 * n - 1);
  const int i0 = (int)f;
  return {i0, min(i0 + 1, n - 1), f - i0};
}
// sigmoid of the bilinear blend of z at (y0, x0) a, (y0, x1) b, (y1, x0) c, (y1, x1) d
__device__ __forceinline__ float up2_sigmoid(float a, float b, float c, float d, float wx, float wy) {
  const float v = (a * (1 - wx) + b * wx) * (1 - wy) + (c * (1 - wx) + d * wx) * wy;
  return 1.f / (1.f + __expf(-v));
}
// last layer: conv1x1 64 -> A (+bias) before the sigmoid; x [B,HW,64] bf16, w [A][64] f32 -> z [B,A,HW] f32 (NCHW like the reference
// output).  gq_head_up2 runs it on the low-resolution map and k_up2_sigmoid finishes the layer.
__global__ void k_head(const bf16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ z, int B, int HW, int A) {
  __shared__ __align__(16) float sw[8 * 64 + 8];
  for (int i = threadIdx.x; i < A * 64; i += blockDim.x) sw[i] = w[i];
  if (threadIdx.x < A) sw[8 * 64 + threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (size_t)B * HW) return;
  int b = p / HW, pix = p % HW;
  float in[64];
  head_load_pixel(x + p * 64, in);
  for (int a = 0; a < A; a++) z[((size_t)b * A + a) * HW + pix] = head_dot(in, sw, a);
}
// q = sigmoid(UpsamplingBilinear2d(2)(z)) on A planes: z [B*A, H, W] f32 -> q [B*A, 2H, 2W] f32 (align_corners=True).
// The network ends with UP2 -> C1 (1x1 conv + bias) -> sigmoid (Modules.py:250-251,281-283); a 1x1 convolution is linear per pixel and the
// bilinear weights sum to one, so C1(UP2(x)) == UP2(C1(x)): the head runs on the 4x smaller map and only its A planes are up-sampled
__global__ void k_up2_sigmoid(const float* __restrict__ z, float* __restrict__ q, int planes, int H, int W) {
  const int OH = 2 * H, OW = 2 * W;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)planes * OH * OW;
  if (i >= n) return;
  const int ow = i % OW, oh = (i / OW) % OH;
  const size_t pl = i / ((size_t)OW * OH);
  const Up2Tap ty = up2_tap(oh, H), tx = up2_tap(ow, W);
  const float* zp = z + pl * H * W;
  q[i] = up2_sigmoid(__ldg(zp + ty.i0 * W + tx.i0), __ldg(zp + ty.i0 * W + tx.i1), __ldg(zp + ty.i1 * W + tx.i0), __ldg(zp + ty.i1 * W + tx.i1), tx.w, ty.w);
}
// max over the Q-map of every image without writing it: CTA (tx, ty, b) evaluates the head on the low-resolution pixels that its
// HM_T x HM_T tile of the up-sampled map reads (z in shared memory) and the tile's A x HM_T x HM_T sigmoids, and raises qmax[b] to their
// maximum with atomicMax on the float bits (exact and order-free: Q-values are >= +0, where the unsigned order of the bits is the float
// order).  The largest sigmoid is taken, not the sigmoid of the largest pre-activation: __expf makes no promise of monotonicity.
// Rows spanned by a tile: the source row f(o) = o (n - 1) / (2n - 1) grows by less than (HM_T - 1) / 2 over the tile, so floor(f) by at
// most HM_T / 2, and with the second tap the tile reads at most HM_T / 2 + 2 rows (columns alike).
constexpr int HM_T = 32, HM_Z = HM_T / 2 + 2;
__global__ void __launch_bounds__(256) k_head_max(const bf16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                  unsigned* __restrict__ qmax_bits, int H, int W, int A) {
  __shared__ __align__(16) float sw[8 * 64 + 8];
  __shared__ float sz[8][HM_Z][HM_Z];
  __shared__ float swarp[8];
  const int b = blockIdx.z, OH = 2 * H, OW = 2 * W;
  const int oy0 = blockIdx.y * HM_T, ox0 = blockIdx.x * HM_T;
  const int th = min(HM_T, OH - oy0), tw = min(HM_T, OW - ox0);
  const int zy0 = up2_tap(oy0, H).i0, zx0 = up2_tap(ox0, W).i0;
  const int zh = up2_tap(oy0 + th - 1, H).i1 - zy0 + 1, zw = up2_tap(ox0 + tw - 1, W).i1 - zx0 + 1;
  for (int i = threadIdx.x; i < A * 64; i += blockDim.x) sw[i] = w[i];
  if (threadIdx.x < A) sw[8 * 64 + threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.x; i < zh * zw; i += blockDim.x) {
    const int ly = i / zw, lx = i % zw;
    float in[64];
    head_load_pixel(x + (((size_t)b * H + zy0 + ly) * W + zx0 + lx) * 64, in);
    for (int a = 0; a < A; a++) sz[a][ly][lx] = head_dot(in, sw, a);
  }
  __syncthreads();
  float m = 0.f;
  for (int i = threadIdx.x; i < A * th * tw; i += blockDim.x) {
    const int a = i / (th * tw), r = i % (th * tw);
    const Up2Tap ty = up2_tap(oy0 + r / tw, H), tx = up2_tap(ox0 + r % tw, W);
    const int y0 = ty.i0 - zy0, y1 = ty.i1 - zy0, x0 = tx.i0 - zx0, x1 = tx.i1 - zx0;
    const float v = up2_sigmoid(sz[a][y0][x0], sz[a][y0][x1], sz[a][y1][x0], sz[a][y1][x1], tx.w, ty.w);
    m = v > m ? v : m;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const float v = __shfl_xor_sync(0xffffffffu, m, o); m = v > m ? v : m; }
  if ((threadIdx.x & 31) == 0) swarp[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); k++) m = swarp[k] > m ? swarp[k] : m;
    atomicMax(qmax_bits + b, __float_as_uint(m));
  }
}
// the Bellman target y = min(1, r + gamma * qmax) in fp32, product and sum rounded separately (no contraction); NaN propagates like
// torch.clamp
__global__ void k_bellman_target(const float* __restrict__ qmax, const float* __restrict__ reward, float gamma, float* __restrict__ y, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float v = __fadd_rn(reward[b], __fmul_rn(gamma, qmax[b]));
  y[b] = v > 1.f ? 1.f : v;
}
// flat arg-max over the A*HW Q-values of every image (Grasping_Agent_multidiscrete.py:295-299): idx = rot*HW + y*W + x
__global__ void __launch_bounds__(1024) k_argmax(const float* __restrict__ q, int n, int* __restrict__ idx, float* __restrict__ val) {
  __shared__ float sv[1024];
  __shared__ int si[1024];
  const float* qb = q + (size_t)blockIdx.x * n;
  float bv = -1.f; int bi = 0;  // Q-values are sigmoids (> 0); ties go to the lowest flat index, like torch.max over the flattened map
  const int n4 = ((size_t)qb % 16 == 0) ? n / 4 : 0;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    float4 v = __ldg((const float4*)qb + i);
    if (v.x > bv) { bv = v.x; bi = 4 * i; }
    if (v.y > bv) { bv = v.y; bi = 4 * i + 1; }
    if (v.z > bv) { bv = v.z; bi = 4 * i + 2; }
    if (v.w > bv) { bv = v.w; bi = 4 * i + 3; }
  }
  for (int i = 4 * n4 + threadIdx.x; i < n; i += blockDim.x) { float v = qb[i]; if (v > bv) { bv = v; bi = i; } }
  sv[threadIdx.x] = bv; si[threadIdx.x] = bi;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) { float ov = sv[threadIdx.x + o]; int oi = si[threadIdx.x + o]; if (ov > sv[threadIdx.x] || (ov == sv[threadIdx.x] && oi < si[threadIdx.x])) { sv[threadIdx.x] = ov; si[threadIdx.x] = oi; } }
    __syncthreads();
  }
  if (threadIdx.x == 0) { idx[blockIdx.x] = si[0]; val[blockIdx.x] = sv[0]; }
}

// Grasp_Agent.transform_observation with normalize=True, jitter_and_noise=False (Grasping_Agent_multidiscrete.py:301-368), batched:
// depth clipped at `thr`, negated, min-max normalised per image; rgb u8 -> [0,1]; output state [B,4,H,W] f32 (r,g,b,depth)
__global__ void k_obs_minmax(const float* __restrict__ depth, int HW, float thr, float* __restrict__ mm) {
  __shared__ float smin[256], smax[256];
  const float* d = depth + (size_t)blockIdx.x * HW;
  float lo = 3.0e38f, hi = -3.0e38f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) { float v = -fminf(d[i], thr); lo = fminf(lo, v); hi = fmaxf(hi, v); }
  smin[threadIdx.x] = lo; smax[threadIdx.x] = hi;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { smin[threadIdx.x] = fminf(smin[threadIdx.x], smin[threadIdx.x + o]); smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + o]); }
    __syncthreads();
  }
  if (threadIdx.x == 0) { mm[2 * blockIdx.x] = smin[0]; mm[2 * blockIdx.x + 1] = smax[0]; }
}
__global__ void k_obs_state(const unsigned char* __restrict__ rgb, const float* __restrict__ depth, const float* __restrict__ mm, float thr, int B, int HW,
                            float* __restrict__ state) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * HW) return;
  int b = i / HW, p = i % HW;
  float lo = mm[2 * b], hi = mm[2 * b + 1];
  float* out = state + (size_t)b * 4 * HW + p;
  out[0] = rgb[3 * i] * (1.f / 255.f); out[HW] = rgb[3 * i + 1] * (1.f / 255.f); out[2 * HW] = rgb[3 * i + 2] * (1.f / 255.f);
  out[3 * (size_t)HW] = (-fminf(depth[i], thr) - lo) / (hi - lo);
}

// ---- training-time transform_observation (normalize=True, jitter_and_noise=True; Grasping_Agent_multidiscrete.py:118-124,301-368):
// depth clipped, + N(0, noise_std) per pixel, negated, min-max normalised per image AFTER the noise (:318-322); rgb through
// ColorJitter(brightness, contrast, saturation, hue) with the per-image factors and operation order drawn by the caller (torchvision's
// get_params: randperm(4) + four uniforms), applied with torchvision's float-tensor arithmetic (_blend / rgb_to_grayscale / _rgb2hsv /
// _hsv2rgb).  The noise comes from a counter-based generator (Philox4x32-10) keyed on the seed and indexed by (global env id, step,
// pixel): the value of a pixel does not depend on how the envs are batched or sharded over GPUs.
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
// standard normal from counter (pixel, env, step) under key = seed (Box-Muller on two of the four words)
__device__ __forceinline__ float obs_noise(uint64_t seed, uint64_t env, uint32_t step, uint32_t pixel) {
  uint32_t w[4];
  philox4x32_10(pixel, (uint32_t)env, (uint32_t)(env >> 32), step, (uint32_t)seed, (uint32_t)(seed >> 32), w);
  const float u1 = ((float)(w[0] >> 8) + 0.5f) * (1.0f / 16777216.0f), u2 = ((float)(w[1] >> 8) + 0.5f) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }
__device__ __forceinline__ float gray_of(float r, float g, float b) { return 0.2989f * r + 0.587f * g + 0.114f * b; }
// one ColorJitter operation on one pixel; op: 0 brightness, 1 contrast (needs the image's grey mean), 2 saturation, 3 hue
__device__ __forceinline__ void jitter_op(int op, float f, float mean, float& r, float& g, float& b) {
  if (op == 0) { r = clamp01(f * r); g = clamp01(f * g); b = clamp01(f * b); }
  else if (op == 1) { const float m = (1.f - f) * mean; r = clamp01(f * r + m); g = clamp01(f * g + m); b = clamp01(f * b + m); }
  else if (op == 2) { const float m = (1.f - f) * gray_of(r, g, b); r = clamp01(f * r + m); g = clamp01(f * g + m); b = clamp01(f * b + m); }
  else {
    const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
    const bool eqc = maxc == minc;
    const float cr = maxc - minc, s = cr / (eqc ? 1.f : maxc), div = eqc ? 1.f : cr;
    const float rc = (maxc - r) / div, gc = (maxc - g) / div, bc = (maxc - b) / div;
    const float hr = (maxc == r) ? (bc - gc) : 0.f, hg = (maxc == g && maxc != r) ? (2.f + rc - bc) : 0.f, hb = (maxc != g && maxc != r) ? (4.f + gc - rc) : 0.f;
    float h = fmodf((hr + hg + hb) / 6.f + 1.f, 1.f);
    h = h + f;                       // torch's % : result has the sign of the divisor
    h = h - floorf(h);
    const float v = maxc, h6 = h * 6.f, fl = floorf(h6), ff = h6 - fl;
    int i = ((int)fl) % 6;
    if (i < 0) i += 6;
    const float pp = clamp01(v * (1.f - s)), q = clamp01(v * (1.f - s * ff)), t = clamp01(v * (1.f - s * (1.f - ff)));
    r = i == 0 ? v : i == 1 ? q : i == 2 ? pp : i == 3 ? pp : i == 4 ? t : v;
    g = i == 0 ? t : i == 1 ? v : i == 2 ? v : i == 3 ? q : i == 4 ? pp : pp;
    b = i == 0 ? pp : i == 1 ? pp : i == 2 ? t : i == 3 ? v : i == 4 ? v : q;
  }
}
// ---- keyed draws: every random decision of the online trainer is a function of (seed, global env, step), like the depth noise.
// Counter (c0, env_lo, env_hi, step), key (seed_lo, seed_hi) of philox4x32_10.  The depth noise uses c0 = pixel < 2^31; the draws below
// use c0 = 0x80000000 + j, so the two streams never overlap:
//   j = 0      w0 -> epsilon uniform u (the transition is greedy iff u > eps); w1, w2, w3 -> brightness, contrast, saturation factors
//   j = 1      w0 -> hue factor; w1 -> operation order = permutation number (uint64)w1 * 24 >> 32 of (0,1,2,3), permutations in
//              lexicographic order (0 = 0123, 1 = 0132, ..., 23 = 3210)
//   j = 2 + k  w0 -> k-th random-action candidate (uint64)w0 * (W*H*R) >> 32 (flat action rot*W*H + y*W + x)
// Prioritized replay (qnet_replay.cuh) draws in its own domain c0 = 0xC0000000 + j, above both of these, with counter
// (c0, update_lo, update_hi, rank): the learner update and the process rank take the place of the env and the step.
//   j < B      w0, w1 -> stratum j's uniform U = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53 in double (53 bits)
// Uniforms are ((w >> 8) + 0.5) / 2^24 in float, as in obs_noise; factors 0.5 + u (brightness, contrast, saturation: 1 +- 0.5) and
// u - 0.5 (hue: +-0.5), the ranges of ColorJitter(0.5, 0.5, 0.5, 0.5).  tests/test_batched_train.py restates this table in numpy.
#define KEYED_C0 0x80000000u
__device__ __forceinline__ void keyed_words(uint64_t seed, uint64_t env, uint32_t step, uint32_t j, uint32_t* w) {
  philox4x32_10(KEYED_C0 + j, (uint32_t)env, (uint32_t)(env >> 32), step, (uint32_t)seed, (uint32_t)(seed >> 32), w);
}
__device__ __forceinline__ float keyed_uniform(uint32_t w) { return ((float)(w >> 8) + 0.5f) * (1.0f / 16777216.0f); }
// the ColorJitter factors (brightness, contrast, saturation, hue) and operation order of one (env, step)
__device__ void keyed_jitter(uint64_t seed, uint64_t env, uint32_t step, float* fac, int* ord) {
  uint32_t w[4], v[4];
  keyed_words(seed, env, step, 0, w);
  keyed_words(seed, env, step, 1, v);
  fac[0] = 0.5f + keyed_uniform(w[1]); fac[1] = 0.5f + keyed_uniform(w[2]); fac[2] = 0.5f + keyed_uniform(w[3]);
  fac[3] = keyed_uniform(v[0]) - 0.5f;
  int p = (int)(((uint64_t)v[1] * 24u) >> 32), left = 0x3210;  // factorial-base digits 6, 2, 1 pick from the unused operations (nibbles)
  const int radix[3] = {6, 2, 1};
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const int d = p / radix[k];
    p -= d * radix[k];
    ord[k] = (left >> (4 * d)) & 15;
    const int lowmask = (1 << (4 * d)) - 1;
    left = (left & lowmask) | ((left >> 4) & ~lowmask);  // drop nibble d
  }
  ord[3] = left & 15;
}

// per image: min / max of the noisy negated clipped depth, and the grey mean of the image as it is when the contrast operation runs.
// Row b reads image slot[b] (NULL: b) and is keyed on env_index[b] (NULL: b) and steps[b] (NULL: step).  With draw_fac / draw_ord
// the row's factors and order are the keyed draws of (seed, env, step), written there for k_obs_train_state; otherwise they come
// from jitter / order.
__global__ void __launch_bounds__(256) k_obs_train_reduce(const unsigned char* __restrict__ rgb, const float* __restrict__ depth, int HW, float thr, float noise_std,
                                                          unsigned long long seed, const long long* __restrict__ slot, const long long* __restrict__ env_index,
                                                          const unsigned int* __restrict__ steps, unsigned int step, const float* __restrict__ jitter,
                                                          const int* __restrict__ order, float* __restrict__ draw_fac, int* __restrict__ draw_ord,
                                                          float* __restrict__ red) {
  __shared__ float smin[256], smax[256];
  __shared__ double ssum[256];
  __shared__ float sfac[4];
  __shared__ int sord[4];
  const int b = blockIdx.x;
  const size_t s = slot ? (size_t)slot[b] : (size_t)b;
  const unsigned long long env = env_index ? (unsigned long long)env_index[b] : (unsigned long long)b;
  if (steps) step = steps[b];
  int ord[4] = {0, 1, 2, 3};
  float fac[4] = {1.f, 1.f, 1.f, 0.f};
  if (draw_fac) {
    if (threadIdx.x == 0) {
      keyed_jitter(seed, env, step, sfac, sord);
      for (int k = 0; k < 4; k++) { draw_fac[4 * b + k] = sfac[k]; draw_ord[4 * b + k] = sord[k]; }
    }
    __syncthreads();
    for (int k = 0; k < 4; k++) { fac[k] = sfac[k]; ord[k] = sord[k]; }
  } else {
    if (jitter) for (int k = 0; k < 4; k++) fac[k] = jitter[4 * b + k];
    if (order) for (int k = 0; k < 4; k++) ord[k] = order[4 * b + k];
  }
  const bool jit = draw_fac || jitter;  // ColorJitter applied (drawn here or given)
  float lo = 3.0e38f, hi = -3.0e38f;
  double gs = 0;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    float v = -(fminf(depth[s * HW + i], thr) + noise_std * obs_noise(seed, env, step, (uint32_t)i));
    lo = fminf(lo, v); hi = fmaxf(hi, v);
    if (jit) {
      const unsigned char* px = rgb + (s * HW + i) * 3;
      float r = px[0] * (1.f / 255.f), g = px[1] * (1.f / 255.f), bl = px[2] * (1.f / 255.f);
      for (int k = 0; k < 4 && ord[k] != 1; k++) jitter_op(ord[k], fac[ord[k]], 0.f, r, g, bl);  // the operations in front of contrast
      gs += gray_of(r, g, bl);
    }
  }
  smin[threadIdx.x] = lo; smax[threadIdx.x] = hi; ssum[threadIdx.x] = gs;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      smin[threadIdx.x] = fminf(smin[threadIdx.x], smin[threadIdx.x + o]); smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + o]);
      ssum[threadIdx.x] += ssum[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { red[4 * b] = smin[0]; red[4 * b + 1] = smax[0]; red[4 * b + 2] = (float)(ssum[0] / HW); red[4 * b + 3] = 0.f; }
}
__global__ void k_obs_train_state(const unsigned char* __restrict__ rgb, const float* __restrict__ depth, const float* __restrict__ red, float thr, float noise_std,
                                  unsigned long long seed, const long long* __restrict__ slot, const long long* __restrict__ env_index,
                                  const unsigned int* __restrict__ steps, unsigned int step, const float* __restrict__ jitter, const int* __restrict__ order, int B,
                                  int HW, float* __restrict__ state, bf16* __restrict__ state_nhwc) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * HW) return;
  const int b = i / HW, p = i % HW;
  const size_t src = (slot ? (size_t)slot[b] : (size_t)b) * HW + p;
  const unsigned long long env = env_index ? (unsigned long long)env_index[b] : (unsigned long long)b;
  if (steps) step = steps[b];
  float r = rgb[3 * src] * (1.f / 255.f), g = rgb[3 * src + 1] * (1.f / 255.f), bl = rgb[3 * src + 2] * (1.f / 255.f);
  if (jitter) {
    const float mean = red[4 * b + 2];
    for (int k = 0; k < 4; k++) { const int op = order ? order[4 * b + k] : k; jitter_op(op, jitter[4 * b + op], mean, r, g, bl); }
  }
  const float lo = red[4 * b], hi = red[4 * b + 1];
  const float d = (-(fminf(depth[src], thr) + noise_std * obs_noise(seed, env, step, (uint32_t)p)) - lo) / (hi - lo);
  if (state) {
    float* out = state + (size_t)b * 4 * HW + p;
    out[0] = r; out[HW] = g; out[2 * (size_t)HW] = bl; out[3 * (size_t)HW] = d;
  }
  if (state_nhwc) {
    __nv_bfloat162* o = (__nv_bfloat162*)(state_nhwc + i * 4);
    o[0] = __floats2bfloat162_rn(r, g); o[1] = __floats2bfloat162_rn(bl, d);
  }
}

// ---- Grasp_Agent.epsilon_greedy (Grasping_Agent_multidiscrete.py:232-282) for a batch, one warp per env.  Greedy iff the keyed
// uniform u > eps[b]; otherwise the reference's rejection sampling: candidate k (keyed draw j = 2 + k) is accepted when its pixel's
// world z >= z_min.  The 32 lanes test candidates 32 at a time and the lowest accepted k wins, which is the first accepted candidate
// of the sequential loop.  After max_draws rejections the last candidate is taken and `exhausted` set.
struct SampleCam { double fovy, pos[3], mat[9]; };
// z of pixel_2_world with the arithmetic of the engine's k_pixel_2_world (grasp_engine.cu): the same expressions, so that the accept
// decisions equal ge_pixel_2_world's
__device__ __forceinline__ double pixel_world_z(const SampleCam& c, int W, int H, int px, int py, float depth) {
  const double PI = 3.14159265358979323846;
  double f = 0.5 * H / tan(c.fovy * PI / 360.0), d = -(double)depth;
  double pc[3] = {(px * d - 0.5 * W * d) / f, (py * d - 0.5 * H * d) / f, d}, t[3];
  t[0] = pc[0] + c.pos[0]; t[1] = pc[1] + c.pos[1]; t[2] = pc[2] + c.pos[2];
  return c.mat[2] * t[0] + c.mat[5] * t[1] + c.mat[8] * t[2];
}
__global__ void __launch_bounds__(256) k_sample_actions(const float* __restrict__ depth, const int* __restrict__ greedy_idx, const double* __restrict__ eps,
                                                        unsigned long long seed, const long long* __restrict__ env_index, unsigned int step, SampleCam cam,
                                                        double z_min, int W, int H, int R, int max_draws, int B, int* __restrict__ action,
                                                        unsigned char* __restrict__ is_random, unsigned char* __restrict__ exhausted) {
  const int b = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const int HW = W * H;
  const unsigned long long env = env_index ? (unsigned long long)env_index[b] : (unsigned long long)b;
  uint32_t w[4];
  keyed_words(seed, env, step, 0, w);
  int flat;
  bool rnd = !(keyed_uniform(w[0]) > eps[b]), none = false;
  if (!rnd) {
    flat = greedy_idx[b];
  } else {
    const float* dimg = depth + (size_t)b * HW;
    const uint32_t n_act = (uint32_t)(HW * R);
    flat = -1;
    for (int base = 0; base < max_draws; base += 32) {
      const int k = base + lane;
      keyed_words(seed, env, step, 2u + (uint32_t)k, w);
      const int cand = (int)(((uint64_t)w[0] * n_act) >> 32), a1 = cand % HW, x = a1 % W, y = a1 / W;
      const bool ok = k < max_draws && pixel_world_z(cam, W, H, x, y, __ldg(dimg + a1)) >= z_min;
      const unsigned acc = __ballot_sync(0xffffffffu, ok);
      if (acc) { flat = __shfl_sync(0xffffffffu, cand, __ffs(acc) - 1); break; }
      if (base + 32 >= max_draws) { flat = __shfl_sync(0xffffffffu, cand, (max_draws - 1) - base); none = true; }
    }
  }
  if (lane == 0) {
    action[2 * b] = flat % HW; action[2 * b + 1] = flat / HW;
    is_random[b] = rnd; exhausted[b] = none;
  }
}

// ------------------------------------------------------------------------------------------------ C-ABI
extern "C" int gq_obs_to_state_train(const unsigned char* rgb, const float* depth, float depth_threshold, float noise_std, unsigned long long seed,
                                     const long long* env_index, unsigned int step, const float* jitter, const int* order, float* scratch_red,
                                     float* state, void* state_nhwc_bf16, int B, int HW, void* stream) {
  if (!rgb || !depth || !scratch_red || (!state && !state_nhwc_bf16) || B <= 0 || HW <= 0) { snprintf(q_err, sizeof q_err, "gq_obs_to_state_train: bad argument"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  k_obs_train_reduce<<<B, 256, 0, st>>>(rgb, depth, HW, depth_threshold, noise_std, seed, nullptr, env_index, nullptr, step, jitter, order, nullptr, nullptr,
                                        scratch_red);
  k_obs_train_state<<<(unsigned)(((size_t)B * HW + 255) / 256), 256, 0, st>>>(rgb, depth, scratch_red, depth_threshold, noise_std, seed, nullptr, env_index, nullptr,
                                                                              step, jitter, order, B, HW, state, (bf16*)state_nhwc_bf16);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_obs_to_state_keyed(const unsigned char* rgb, const float* depth, const long long* slot, const long long* env_index, const unsigned int* step,
                                     float depth_threshold, float noise_std, unsigned long long seed, float* scratch_red, float* jitter_out, int* order_out,
                                     float* state, void* state_nhwc_bf16, int B, int HW, void* stream) {
  if (!rgb || !depth || !env_index || !step || !scratch_red || !jitter_out || !order_out || (!state && !state_nhwc_bf16) || B <= 0 || HW <= 0) {
    snprintf(q_err, sizeof q_err, "gq_obs_to_state_keyed: bad argument");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  k_obs_train_reduce<<<B, 256, 0, st>>>(rgb, depth, HW, depth_threshold, noise_std, seed, slot, env_index, step, 0u, nullptr, nullptr, jitter_out, order_out,
                                        scratch_red);
  k_obs_train_state<<<(unsigned)(((size_t)B * HW + 255) / 256), 256, 0, st>>>(rgb, depth, scratch_red, depth_threshold, noise_std, seed, slot, env_index, step,
                                                                              0u, jitter_out, order_out, B, HW, state, (bf16*)state_nhwc_bf16);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_sample_actions(const float* depth, const int* greedy_idx, const double* eps, unsigned long long seed, const long long* env_index,
                                 unsigned int step, double fovy, const double* cam_pos, const double* cam_mat, double z_min, int W, int H, int R, int max_draws,
                                 int B, int* action, unsigned char* is_random, unsigned char* exhausted, void* stream) {
  if (!depth || !greedy_idx || !eps || !env_index || !cam_pos || !cam_mat || !action || !is_random || !exhausted || W <= 0 || H <= 0 || R <= 0 ||
      max_draws <= 0 || B <= 0 || (long long)W * H * R > 0x7fffffffLL) {
    snprintf(q_err, sizeof q_err, "gq_sample_actions: bad argument");
    return -1;
  }
  SampleCam cam;
  cam.fovy = fovy;
  for (int k = 0; k < 3; k++) cam.pos[k] = cam_pos[k];
  for (int k = 0; k < 9; k++) cam.mat[k] = cam_mat[k];
  k_sample_actions<<<(unsigned)(((size_t)B * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(depth, greedy_idx, eps, seed, env_index, step, cam, z_min, W, H, R,
                                                                                                max_draws, B, action, is_random, exhausted);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_obs_to_state(const unsigned char* rgb, const float* depth, float depth_threshold, float* scratch_minmax, float* state, int B, int HW,
                               void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  k_obs_minmax<<<B, 256, 0, st>>>(depth, HW, depth_threshold, scratch_minmax);
  k_obs_state<<<(unsigned)(((size_t)B * HW + 255) / 256), 256, 0, st>>>(rgb, depth, scratch_minmax, depth_threshold, B, HW, state);
  QCK(cudaGetLastError());
  return 0;
}

extern "C" const char* gq_version(void) { return "grasp_qnet 0.7 sm_90a bf16 wgmma (persistent CTAs, both operands by TMA: im2col activations + tiled weights, SW128 K-major, register accumulators, fused block tail, BN-folded dual-source eval blocks)"; }

// tile shape: 128 output pixels x 128 output channels (64 when 128 does not divide Cout); the accumulator of a consumer warpgroup is
// 64 x BLOCK_N fp32 = BLOCK_N / 2 registers per thread.  One CTA per SM with 192 KB of stages (6 at BLOCK_N 128, 8 at 64): on an H100
// (700 W) the whole forward ran at 297 TFLOP/s this way against 287 with two CTAs per SM of 96 KB each, whose 96-register cap spilled.
static int conv_block_n(int Cout) { return (Cout % 128 == 0) ? 128 : 64; }
static size_t conv_smem(int bn, int nst) { return 1024 + (size_t)nst * (BM * BK * 2 + (size_t)bn * BK * 2) + 16 * (size_t)nst; }

// 2-D tensor map of the packed weights w [Cout][taps * Cin] bf16 with a [BLOCK_N rows x 64 columns] box, 128-byte swizzle (the layout the
// wgmma descriptors expect); cuTensorMapEncodeTiled comes from the driver through the runtime (no libcuda link dependency)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int make_weight_tmap(CUtensorMap* m, const void* w, int Cout, int K, int bn) {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
  }
  if (!fn) { snprintf(q_err, sizeof q_err, "cuTensorMapEncodeTiled is not available"); return -3; }
  cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)Cout};
  cuuint64_t gstride[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)bn};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(q_err, sizeof q_err, "cuTensorMapEncodeTiled failed (%d)", (int)r); return -3; }
  return 0;
}

// im2col-mode tensor map of the activations x [N][H][W][C] bf16: 64 channels x 128 output positions per load, zero fill outside the image
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*, const int*,
                                   cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);
static int make_act_tmap_im2col(CUtensorMap* m, const void* x, int B, int H, int W, int C, int ks) {
  static EncodeIm2colFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess) fn = (EncodeIm2colFn)p;
  }
  if (!fn) { snprintf(q_err, sizeof q_err, "cuTensorMapEncodeIm2col is not available"); return -3; }
  const int pad = ks / 2;
  cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t gstride[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  int lower[2] = {-pad, -pad}, upper[2] = {pad - (ks - 1), pad - (ks - 1)};  // fprop corners (W, H): as many box positions as output pixels
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), gdim, gstride, lower, upper, (cuuint32_t)BK, (cuuint32_t)BM, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(q_err, sizeof q_err, "cuTensorMapEncodeIm2col failed (%d)", (int)r); return -3; }
  return 0;
}

// EPI 0: y (+ BN partials); EPI 1: out = relu(resid * scale + shift + conv + bias) bf16; EPI 2: out = [relu](conv + bias) bf16.
// grid = (m tiles, n tiles, images) of the problem.  x2 / Cx: optional second source, a 1x1 convolution appended to the K loop.
template <int EPI>
static int launch_conv(int bn, dim3 grid, cudaStream_t st, const bf16* x, const bf16* w, const float* bias, float* y, float* partials,
                       const float* resid, const float2* ss, bf16* out, int H, int W, int Cin, int Cout, int ks, const bf16* x2 = nullptr, int Cx = 0,
                       int relu = 0) {
  alignas(64) CUtensorMap tm, tmx, tmx2;
  memset(&tm, 0, sizeof tm);
  memset(&tmx, 0, sizeof tmx);
  memset(&tmx2, 0, sizeof tmx2);
  int r = make_weight_tmap(&tm, w, Cout, ks * ks * Cin + Cx, bn);
  if (r == 0) r = make_act_tmap_im2col(&tmx, x, (int)grid.z, H, W, Cin, ks);
  if (r == 0 && Cx > 0) r = make_act_tmap_im2col(&tmx2, x2, (int)grid.z, H, W, Cx, 1);
  if (r) return r;
  int dev = 0, sms = 0;
  QCK(cudaGetDevice(&dev));
  QCK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int gx = (int)grid.x, gy = (int)grid.y, ntiles = gx * gy * (int)grid.z;
  const int nctas = ntiles < sms ? ntiles : sms;
#define LAUNCH_T(BN_, ST_)                                                                                                             \
  do {                                                                                                                                 \
    const size_t smem = conv_smem(BN_, ST_);                                                                                           \
    QCK(cudaFuncSetAttribute(k_conv_wgmma<BN_, ST_, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                     \
    k_conv_wgmma<BN_, ST_, EPI><<<nctas, CONV_THREADS, smem, st>>>(tm, tmx, tmx2, bias, y, partials, resid, ss, out, H, W, Cin, Cx, Cout, ks, relu, gx, gy, \
                                                                   ntiles);                                                            \
  } while (0)
  if (bn == 128) LAUNCH_T(128, 6);
  else LAUNCH_T(64, 8);
#undef LAUNCH_T
  return 0;
}

extern "C" size_t gq_conv_partials_floats(int B, int H, int W, int Cout) {
  return (size_t)B * ((H * W + BM - 1) / BM) * CONV_PARTS * Cout * 2;
}
extern "C" int gq_conv_tc(const void* x, const void* w, const float* bias, float* y, float* stats, float* partials, int B, int H, int W, int Cin, int Cout, int ks,
                          void* stream) {
  if (!x || !w || !y || (ks != 1 && ks != 3) || Cin % 64 || Cout % 64) { snprintf(q_err, sizeof q_err, "gq_conv_tc: bad argument"); return -1; }
  if (stats && !partials) { snprintf(q_err, sizeof q_err, "gq_conv_tc: stats requested without a partials buffer"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  const int bn = conv_block_n(Cout);
  dim3 grid((H * W + BM - 1) / BM, Cout / bn, B);
  int r = launch_conv<0>(bn, grid, st, (const bf16*)x, (const bf16*)w, bias, y, stats ? partials : nullptr, nullptr, nullptr, nullptr, H, W, Cin, Cout, ks);
  if (r) return r;
  if (stats) k_bn_reduce<<<(B * Cout + 127) / 128, 128, 0, st>>>(partials, stats, B, (int)grid.x * CONV_PARTS, Cout);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_conv_tc_block_out(const void* x, const void* w, const float* bias, const float* resid, const float* stats, const float* gamma,
                                    const float* beta, float eps, float* scratch_scale_shift, void* out, int B, int H, int W, int Cin, int Cout, int ks,
                                    void* stream) {
  if (!x || !w || !resid || !stats || !gamma || !beta || !scratch_scale_shift || !out || (ks != 1 && ks != 3) || Cin % 64 || Cout % 64) {
    snprintf(q_err, sizeof q_err, "gq_conv_tc_block_out: bad argument");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int bn = conv_block_n(Cout);
  dim3 grid((H * W + BM - 1) / BM, Cout / bn, B);
  k_bn_scale_shift<<<(B * Cout + 127) / 128, 128, 0, st>>>(stats, gamma, beta, (float2*)scratch_scale_shift, B, Cout, H * W, eps);
  int r = launch_conv<1>(bn, grid, st, (const bf16*)x, (const bf16*)w, bias, nullptr, nullptr, resid, (const float2*)scratch_scale_shift, (bf16*)out, H, W, Cin, Cout, ks);
  if (r) return r;
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_conv_tc_fused(const void* a, const void* x, const void* w, const float* bias, void* out, int relu, int B, int H, int W, int Ca, int Cx,
                                int Cout, int ks_a, void* stream) {
  if (!a || !w || !out || (ks_a != 1 && ks_a != 3) || Ca <= 0 || Ca % 64 || Cout <= 0 || Cout % 64 || Cx < 0 || Cx % 64 || (Cx > 0) != (x != nullptr) || B <= 0) {
    snprintf(q_err, sizeof q_err, "gq_conv_tc_fused: bad argument");
    return -1;
  }
  const int bn = conv_block_n(Cout);
  dim3 grid((H * W + BM - 1) / BM, Cout / bn, B);
  int r = launch_conv<2>(bn, grid, (cudaStream_t)stream, (const bf16*)a, (const bf16*)w, bias, nullptr, nullptr, nullptr, nullptr, (bf16*)out, H, W, Ca, Cout, ks_a,
                         (const bf16*)x, Cx, relu ? 1 : 0);
  if (r) return r;
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_conv_first(const float* x, const float* w, void* y, int B, int H, int W, void* stream) {
  k_conv_first2<<<((B * H * W + 1) / 2 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(x, w, (bf16*)y, B, H, W);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_maxpool(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  size_t n = (size_t)B * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
  k_maxpool<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)y, B, H, W, C);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_bn_act(const float* x, const float* stats, const float* gamma, const float* beta, const float* identity, void* y, int B, int HW, int C,
                         float eps, void* stream) {
  if (C % 8) { snprintf(q_err, sizeof q_err, "gq_bn_act: C must be a multiple of 8"); return -1; }
  // enough CTAs per image to fill the GPU (8 per SM) without making the per-CTA prologue (2 C floats) matter
  int dev = 0, sms = 0;
  QCK(cudaGetDevice(&dev));
  QCK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int ctas = (sms * 8 + B - 1) / B;
  int ppc = (HW + ctas - 1) / ctas;
  if (ppc < 16) ppc = 16;
  dim3 grid((HW + ppc - 1) / ppc, B);
  k_bn_act<<<grid, 256, 2 * C * sizeof(float), (cudaStream_t)stream>>>(x, stats, gamma, beta, identity, (bf16*)y, HW, C, eps, ppc);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_upsample2x(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  if (C % 8) { snprintf(q_err, sizeof q_err, "gq_upsample2x: C must be a multiple of 8"); return -1; }
  size_t n = (size_t)B * 4 * H * W * (C / 8);
  k_upsample2x<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)y, B, H, W, C);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_head_up2(const void* x, const float* w, const float* bias, float* scratch_z, float* q, int B, int H, int W, int A, void* stream) {
  if (A > 8 || !scratch_z) { snprintf(q_err, sizeof q_err, "gq_head_up2: bad argument"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  k_head<<<(unsigned)(((size_t)B * H * W + 127) / 128), 128, 0, st>>>((const bf16*)x, w, bias, scratch_z, B, H * W, A);
  size_t n = (size_t)B * A * 4 * H * W;
  k_up2_sigmoid<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(scratch_z, q, B * A, H, W);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_head_max_target(const void* x, const float* w, const float* bias, const float* reward, float gamma, float* qmax, float* y, int B, int H,
                                  int W, int A, void* stream) {
  if (A < 1 || A > 8 || B < 1 || H < 1 || W < 1 || B > 65535) { snprintf(q_err, sizeof q_err, "gq_head_max_target: bad argument"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  QCK(cudaMemsetAsync(qmax, 0, (size_t)B * sizeof(float), st));  // +0.0f: below every sigmoid value
  k_head_max<<<dim3((2 * W + HM_T - 1) / HM_T, (2 * H + HM_T - 1) / HM_T, B), 256, 0, st>>>((const bf16*)x, w, bias, (unsigned*)qmax, H, W, A);
  k_bellman_target<<<(B + 127) / 128, 128, 0, st>>>(qmax, reward, gamma, y, B);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_argmax(const float* q, int B, int n, int* idx, float* val, void* stream) {
  k_argmax<<<B, 1024, 0, (cudaStream_t)stream>>>(q, n, idx, val);
  QCK(cudaGetLastError());
  return 0;
}
#include "qnet_learn.cuh"
#include "qnet_replay.cuh"
