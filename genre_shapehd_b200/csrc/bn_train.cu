// bn_train.cu — BatchNorm3d with batch statistics (training mode) fused with its LeakyReLU/ReLU, forward and backward,
// for NCDHW fp32 activations: the normalisation blocks of Conv3d_block / Deconv3d_skip (networks/networks.py:193-222) and
// of the decoders' deconv stacks (:40-57) while training.
//
// Why: after the convolution fixes of this round a Unet_3D training step at B=4 spends 4.0 ms in cuDNN's
// bn_bw_1C11_kernel_new and 1.3 ms in bn_fw_tr_1C11_kernel_NCHW (profiles/r01_train_unet_launches.csv) for tensors whose
// HBM traffic is worth ~0.05 ms each, plus separate LeakyReLU passes.  These kernels are pure streaming reductions +
// elementwise maps: HBM-bound, float4 accesses, a (split, channel) grid sized for the SM count, two-pass variance (no
// E[x^2] - E[x]^2 cancellation), fixed-order reductions (bitwise reproducible).
//
//   forward : sum -> mean;  sum (x - mean)^2 -> biased var;  y = act(gamma * (x - mean) * invstd + beta)
//             running_mean/var updated with momentum (unbiased var), mean / invstd saved for the backward
//   backward: g = dy * act'(pre);  dbeta = sum g;  dgamma = sum g * xhat;
//             dx = gamma * invstd * (g - dbeta / N - xhat * dgamma / N)
//
// The pre-activation is formed by ONE helper, bn_pre(), in the forward and in both backward kernels: the backward's
// activation mask is then exactly the sign of what the forward computed (autograd differentiates what ran), and x == mean
// with beta == 0 gives exactly 0.  Routed by default for training-mode BatchNorm3d (ops_conv.BN_TRAIN,
// GENRE_B200_BN_TRAIN=0 turns it off); tests/test_gpu_train_fp64.py checks it against an fp64 reference.
#include "common.cuh"

namespace gb {

constexpr int BN_THREADS = 256;
constexpr int BN_MAX_SPLIT = 64;

struct BnShape {
  int B, C;
  long long S;      // D*H*W, a multiple of 4
  int nsplit;       // CTAs per channel
  long long chunk;  // float4 elements of one (b, c) row handled per CTA = ceil(S/4 / nsplit)
};

__device__ __forceinline__ float block_sum(float v, float *s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float t = 0.0f;
  if (warp == 0) {
    t = lane < BN_THREADS / 32 ? s_red[lane] : 0.0f;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  return t;  // valid in warp 0 (all its lanes)
}

// fixed-order total of the per-split partials of channel c
__device__ __forceinline__ float total_of(const float *__restrict__ partial, int c, int nsplit) {
  float t = 0.0f;
  for (int s = 0; s < nsplit; ++s) t += partial[(size_t)c * BN_MAX_SPLIT + s];
  return t;
}

// iterate this CTA's float4 elements of channel c: f(b, i4) with i4 in [lo, hi)
template <typename F>
__device__ __forceinline__ void for_each_vec(const BnShape &sh, int split, F f) {
  const long long n4 = sh.S / 4;
  const long long lo = (long long)split * sh.chunk, hi = min(n4, lo + sh.chunk);
  for (int b = 0; b < sh.B; ++b)
    for (long long i = lo + threadIdx.x; i < hi; i += BN_THREADS) f(b, i);
}

// pass 1: partial sums of x
__global__ void __launch_bounds__(BN_THREADS)
bn_sum_kernel(const float4 *__restrict__ x, BnShape sh, float *__restrict__ psum) {
  __shared__ float s_red[BN_THREADS / 32];
  const int split = blockIdx.x, c = blockIdx.y;
  const long long n4 = sh.S / 4;
  float acc = 0.0f;
  for_each_vec(sh, split, [&](int b, long long i) {
    const float4 v = __ldg(x + ((size_t)b * sh.C + c) * n4 + i);
    acc += (v.x + v.y) + (v.z + v.w);
  });
  const float t = block_sum(acc, s_red);
  if (threadIdx.x == 0) psum[(size_t)c * BN_MAX_SPLIT + split] = t;
}

// pass 2: partial sums of (x - mean)^2
__global__ void __launch_bounds__(BN_THREADS)
bn_sqdev_kernel(const float4 *__restrict__ x, BnShape sh, const float *__restrict__ psum, float *__restrict__ psq) {
  __shared__ float s_red[BN_THREADS / 32];
  const int split = blockIdx.x, c = blockIdx.y;
  const long long n4 = sh.S / 4;
  const float mean = total_of(psum, c, sh.nsplit) / ((float)sh.B * (float)sh.S);
  float acc = 0.0f;
  for_each_vec(sh, split, [&](int b, long long i) {
    const float4 v = __ldg(x + ((size_t)b * sh.C + c) * n4 + i);
    const float a = v.x - mean, bq = v.y - mean, cq = v.z - mean, d = v.w - mean;
    acc += (a * a + bq * bq) + (cq * cq + d * d);
  });
  const float t = block_sum(acc, s_red);
  if (threadIdx.x == 0) psq[(size_t)c * BN_MAX_SPLIT + split] = t;
}

__device__ __forceinline__ float act_fwd(float v, float slope) { return v > 0.0f ? v : v * slope; }

// normalised value and pre-activation in the order of torch's CUDA BatchNorm, ((x - mean) * invstd) * gamma + beta
__device__ __forceinline__ float bn_xhat(float x, float mean, float invstd) { return (x - mean) * invstd; }
__device__ __forceinline__ float bn_pre(float xh, float gamma, float beta) { return fmaf(xh, gamma, beta); }

// pass 3: normalise + affine + activation; split 0 also publishes mean / invstd and updates the running statistics
__global__ void __launch_bounds__(BN_THREADS)
bn_apply_kernel(const float4 *__restrict__ x, BnShape sh, const float *__restrict__ psum, const float *__restrict__ psq,
                const float *__restrict__ gamma, const float *__restrict__ beta, float eps, float momentum, float slope,
                float4 *__restrict__ y, float *__restrict__ save_mean, float *__restrict__ save_invstd,
                float *__restrict__ running_mean, float *__restrict__ running_var) {
  const int split = blockIdx.x, c = blockIdx.y;
  const long long n4 = sh.S / 4;
  const float n = (float)sh.B * (float)sh.S;
  const float mean = total_of(psum, c, sh.nsplit) / n;
  const float var = total_of(psq, c, sh.nsplit) / n;
  const float invstd = rsqrtf(var + eps);
  const float g = gamma ? gamma[c] : 1.0f, bt = beta ? beta[c] : 0.0f;
  if (split == 0 && threadIdx.x == 0) {
    save_mean[c] = mean;
    save_invstd[c] = invstd;
    if (running_mean) running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * mean;
    if (running_var) running_var[c] = (1.0f - momentum) * running_var[c] + momentum * var * (n / fmaxf(n - 1.0f, 1.0f));
  }
  for_each_vec(sh, split, [&](int b, long long i) {
    const size_t at = ((size_t)b * sh.C + c) * n4 + i;
    const float4 v = __ldg(x + at);
    float4 o;
    o.x = act_fwd(bn_pre(bn_xhat(v.x, mean, invstd), g, bt), slope);
    o.y = act_fwd(bn_pre(bn_xhat(v.y, mean, invstd), g, bt), slope);
    o.z = act_fwd(bn_pre(bn_xhat(v.z, mean, invstd), g, bt), slope);
    o.w = act_fwd(bn_pre(bn_xhat(v.w, mean, invstd), g, bt), slope);
    y[at] = o;
  });
}

// backward pass 1: partial sums of g = dy * act'(pre) and of g * xhat
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_sum_kernel(const float4 *__restrict__ x, const float4 *__restrict__ dy, BnShape sh, const float *__restrict__ mean_,
                  const float *__restrict__ invstd_, const float *__restrict__ gamma, const float *__restrict__ beta,
                  float slope, float *__restrict__ pg, float *__restrict__ pgx) {
  __shared__ float s_red[BN_THREADS / 32];
  const int split = blockIdx.x, c = blockIdx.y;
  const long long n4 = sh.S / 4;
  const float mean = mean_[c], invstd = invstd_[c];
  const float g0 = gamma ? gamma[c] : 1.0f, bt = beta ? beta[c] : 0.0f;
  float a0 = 0.0f, a1 = 0.0f;
  for_each_vec(sh, split, [&](int b, long long i) {
    const size_t at = ((size_t)b * sh.C + c) * n4 + i;
    const float4 v = __ldg(x + at), d = __ldg(dy + at);
    const float xv[4] = {v.x, v.y, v.z, v.w}, dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xh = bn_xhat(xv[k], mean, invstd);
      const float pre = bn_pre(xh, g0, bt);
      const float gk = pre > 0.0f ? dv[k] : dv[k] * slope;
      a0 += gk;
      a1 = fmaf(gk, xh, a1);
    }
  });
  const float t0 = block_sum(a0, s_red);
  const float t1 = block_sum(a1, s_red);
  if (threadIdx.x == 0) {
    pg[(size_t)c * BN_MAX_SPLIT + split] = t0;
    pgx[(size_t)c * BN_MAX_SPLIT + split] = t1;
  }
}

// backward pass 2: dx; split 0 publishes dgamma / dbeta
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_apply_kernel(const float4 *__restrict__ x, const float4 *__restrict__ dy, BnShape sh, const float *__restrict__ mean_,
                    const float *__restrict__ invstd_, const float *__restrict__ gamma, const float *__restrict__ beta,
                    float slope, const float *__restrict__ pg, const float *__restrict__ pgx, float4 *__restrict__ dx,
                    float *__restrict__ dgamma, float *__restrict__ dbeta) {
  const int split = blockIdx.x, c = blockIdx.y;
  const long long n4 = sh.S / 4;
  const float n = (float)sh.B * (float)sh.S;
  const float mean = mean_[c], invstd = invstd_[c];
  const float g0 = gamma ? gamma[c] : 1.0f, bt = beta ? beta[c] : 0.0f;
  const float sg = total_of(pg, c, sh.nsplit), sgx = total_of(pgx, c, sh.nsplit);
  if (split == 0 && threadIdx.x == 0) {
    if (dgamma) dgamma[c] = sgx;
    if (dbeta) dbeta[c] = sg;
  }
  const float k0 = g0 * invstd, m0 = sg / n, m1 = sgx / n;
  for_each_vec(sh, split, [&](int b, long long i) {
    const size_t at = ((size_t)b * sh.C + c) * n4 + i;
    const float4 v = __ldg(x + at), d = __ldg(dy + at);
    const float xv[4] = {v.x, v.y, v.z, v.w}, dv[4] = {d.x, d.y, d.z, d.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xh = bn_xhat(xv[k], mean, invstd);
      const float pre = bn_pre(xh, g0, bt);
      const float gk = pre > 0.0f ? dv[k] : dv[k] * slope;
      o[k] = k0 * (gk - m0 - xh * m1);
    }
    dx[at] = make_float4(o[0], o[1], o[2], o[3]);
  });
}

static int bn_shape(int64_t B, int64_t C, int64_t S, BnShape *sh) {
  GB_REQUIRE(B > 0 && C > 0 && S > 0 && S % 4 == 0 && B < (1 << 20) && C < 65536, GENRE_B200_EINVAL,
             "batchnorm: unsupported shape (spatial size must be a multiple of 4)");
  sh->B = (int)B;
  sh->C = (int)C;
  sh->S = S;
  // enough CTAs for ~4 waves of the SMs, at least ~4096 float4 per CTA and batch row
  long long want = ((long long)sm_count() * 4 + C - 1) / C;
  const long long n4 = S / 4;
  long long cap = (n4 + 1023) / 1024;
  long long ns = want < cap ? want : cap;
  if (ns < 1) ns = 1;
  if (ns > BN_MAX_SPLIT) ns = BN_MAX_SPLIT;
  sh->nsplit = (int)ns;
  sh->chunk = (n4 + ns - 1) / ns;
  return 0;
}

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_bn_workspace_bytes(int64_t C) { return (size_t)(C > 0 ? C : 0) * BN_MAX_SPLIT * 2 * sizeof(float); }

// y = act(batchnorm(x)) with batch statistics.  x, y [B][C][S] fp32 contiguous, 16-byte aligned, S % 4 == 0; gamma, beta [C]
// or NULL; running_mean / running_var [C] or NULL (updated in place with `momentum`); save_mean, save_invstd [C] out;
// slope: LeakyReLU slope (1 = no activation, 0 = ReLU); workspace of genre_b200_bn_workspace_bytes(C) bytes.
extern "C" int genre_b200_bn_act_train_forward(const float *x, int64_t B, int64_t C, int64_t S, const float *gamma,
                                               const float *beta, float *running_mean, float *running_var, float eps,
                                               float momentum, float slope, float *y, float *save_mean, float *save_invstd,
                                               void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(x && y && save_mean && save_invstd && workspace, GENRE_B200_EINVAL, "bn_act_train_forward: null pointer");
  GB_REQUIRE(aligned16(x) && aligned16(y), GENRE_B200_EALIGN, "bn_act_train_forward: x and y must be 16-byte aligned");
  GB_REQUIRE(workspace_bytes >= genre_b200_bn_workspace_bytes(C), GENRE_B200_EWORKSPACE, "bn_act_train_forward: workspace too small");
  BnShape sh;
  if (int rc = bn_shape(B, C, S, &sh)) return rc;
  float *psum = (float *)workspace, *psq = psum + (size_t)C * BN_MAX_SPLIT;
  cudaStream_t st = as_stream(stream);
  dim3 grid((unsigned)sh.nsplit, (unsigned)C);
  bn_sum_kernel<<<grid, BN_THREADS, 0, st>>>((const float4 *)x, sh, psum);
  bn_sqdev_kernel<<<grid, BN_THREADS, 0, st>>>((const float4 *)x, sh, psum, psq);
  bn_apply_kernel<<<grid, BN_THREADS, 0, st>>>((const float4 *)x, sh, psum, psq, gamma, beta, eps, momentum, slope, (float4 *)y,
                                               save_mean, save_invstd, running_mean, running_var);
  return check_launch("bn_act_train forward kernels");
}

// dx (and dgamma, dbeta [C], either may be NULL) from dy, the forward's input x and its saved mean / invstd.
extern "C" int genre_b200_bn_act_train_backward(const float *x, const float *dy, int64_t B, int64_t C, int64_t S,
                                                const float *gamma, const float *beta, const float *save_mean,
                                                const float *save_invstd, float slope, float *dx, float *dgamma,
                                                float *dbeta, void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(x && dy && dx && save_mean && save_invstd && workspace, GENRE_B200_EINVAL, "bn_act_train_backward: null pointer");
  GB_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(dx), GENRE_B200_EALIGN, "bn_act_train_backward: alignment");
  GB_REQUIRE(workspace_bytes >= genre_b200_bn_workspace_bytes(C), GENRE_B200_EWORKSPACE, "bn_act_train_backward: workspace too small");
  BnShape sh;
  if (int rc = bn_shape(B, C, S, &sh)) return rc;
  float *pg = (float *)workspace, *pgx = pg + (size_t)C * BN_MAX_SPLIT;
  cudaStream_t st = as_stream(stream);
  dim3 grid((unsigned)sh.nsplit, (unsigned)C);
  bn_bwd_sum_kernel<<<grid, BN_THREADS, 0, st>>>((const float4 *)x, (const float4 *)dy, sh, save_mean, save_invstd, gamma, beta,
                                                 slope, pg, pgx);
  bn_bwd_apply_kernel<<<grid, BN_THREADS, 0, st>>>((const float4 *)x, (const float4 *)dy, sh, save_mean, save_invstd, gamma,
                                                   beta, slope, pg, pgx, (float4 *)dx, dgamma, dbeta);
  return check_launch("bn_act_train backward kernels");
}
