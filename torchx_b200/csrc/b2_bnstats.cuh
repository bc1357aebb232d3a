// b2_bnstats.cuh — the statistics exchange of SyncBatchNorm (b2_batchnorm_stats): every rank's (mean[C], invstd[C], count)
// row is gathered and merged into the global mean / invstd, with the arithmetic of ATen's
// batch_norm_reduce_statistics_kernel<float, float, int32_t> (torch/include/ATen/native/cuda/Normalization.cuh:459-502,
// the kernel behind torch.batch_norm_gather_stats_with_counts) in ATen's order, so the result is the same bits as torch's
// SyncBatchNorm forward.  Every rounding point is written out (DESIGN.md 2.4): nvcc's FMA contraction is not relied upon.
//
// One-shot on ONE CTA: the CTA pushes its row as raw fp32 16-byte vecs into recv[me] of every rank's stage, runs one
// cta_xbar, and merges the W rows out of its own stage.  cta_xbar only orders CTAs with the same blockIdx.x across ranks;
// with a single CTA, the CTA that merges channel i is the one whose barrier covered every rank's whole row, count included.
// A BatchNorm layer has at most a few thousand channels, so a row is a few KiB and one CTA of kThreads threads holds it in
// a handful of vecs per thread.  The op counter, stage parity and flag sequence are those of every other collective.
#pragma once

#include "b2_dev.cuh"
#include "b2_exact.cuh"

namespace bnstats {

// One rank's contribution merged into the running (avg, var_n) of one channel.  n is the float of ATen's integer count so
// far, cnt this rank's count, factor = 1 / (n + cnt) and nfac / cfac = n * factor / cnt * factor (the same for every
// channel).  ATen's source: v = 1/invstd; v = (v*v - eps) * count; var_n += v + (avg-m)*(avg-m)*n*count*factor;
// avg = n*factor*avg + count*factor*m.  Its SASS fuses v*v - eps, the multiply by count into the add of the second term,
// and n*factor*avg into the add of count*factor*m; everything else is rounded on its own.
__device__ __forceinline__ void merge(float& avg, float& var_n, float m, float is, float nf, float cnt, float factor, float nfac,
                                      float cfac, float eps) {
  const float v = __frcp_rn(is);
  const float a = __fmaf_rn(v, v, -eps);
  const float d = __fsub_rn(avg, m);
  const float t = __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), nf), cnt), factor);
  var_n = __fadd_rn(var_n, __fmaf_rn(a, cnt, t));
  avg = __fmaf_rn(nfac, avg, __fmul_rn(m, cfac));
}

__device__ __forceinline__ float lane(const uint4& q, int k) {
  return __uint_as_float(k == 0 ? q.x : (k == 1 ? q.y : (k == 2 ? q.z : q.w)));
}

}  // namespace bnstats

// In place: mean[i] / invstd[i] <- the merge of every rank's (mean, invstd, count) over the ranks with count >= 1, in rank
// order; running_mean / running_var updated when non-null; counts_out[r] <- rank r's count when non-null.  C channels.
// Launched with ONE CTA.  At W = 1 the merge runs on this rank's row alone: no push, no barrier, no op counter.
__global__ void __launch_bounds__(kThreads, 1)
    k_bn_stats(CommDev c, float* mean, float* invstd, float count, unsigned long long C, float* running_mean, float* running_var,
               float momentum, float eps, float* counts_out) {
  using namespace dev;
  const bool solo = c.world == 1;
  uint8_t* pm = reinterpret_cast<uint8_t*>(mean);
  uint8_t* pi = reinterpret_cast<uint8_t*>(invstd);
  const bool am = (reinterpret_cast<uintptr_t>(mean) & 15u) == 0;
  const bool ai = (reinterpret_cast<uintptr_t>(invstd) & 15u) == 0;
  const unsigned long long Cv = (C + 3) / 4;  // vecs of one statistic; the row is mean, invstd, then the count's vec
  uint64_t seq0 = 0;
  const uint8_t* mine = nullptr;
  if (!solo) {
    seq0 = op_begin(c);
    const unsigned long long stage = stage_of(c, seq0);
    for (unsigned long long v = threadIdx.x; v <= 2 * Cv; v += kThreads) {
      uint4 q;
      if (v < Cv) q = exact::ld_local<4>(pm, am, v, C);
      else if (v < 2 * Cv) q = exact::ld_local<4>(pi, ai, v - Cv, C);
      else q = make_uint4(__float_as_uint(count), 0u, 0u, 0u);
      exact::push_vec(c, stage, v, q);
    }
    cta_xbar(c, seq0 * 4u + 1u);
    mine = c.peer[0] + stage;
  }
  // counts in rank order; a rank below one sample is left out of the merge (torch's mask count_all >= 1)
  float cnts[B2_MAX_WORLD];
#pragma unroll
  for (int r = 0; r < B2_MAX_WORLD; ++r)
    cnts[r] = r >= c.world ? 0.0f : (solo ? count : __uint_as_float(ldg_u4(mine + r * c.slice_cap + 2 * Cv * 16).x));
  if (counts_out != nullptr && threadIdx.x < c.world) {
#pragma unroll
    for (int r = 0; r < B2_MAX_WORLD; ++r)
      if (r == static_cast<int>(threadIdx.x)) counts_out[r] = cnts[r];
  }
  const float om = __fsub_rn(1.0f, momentum);
  for (unsigned long long v = threadIdx.x; v < Cv; v += kThreads) {
    float avg[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    float var_n[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    int n = 0;
#pragma unroll
    for (int r = 0; r < B2_MAX_WORLD; ++r) {
      if (r >= c.world || !(cnts[r] >= 1.0f)) continue;
      uint4 qm, qi;
      if (solo) {
        qm = exact::ld_local<4>(pm, am, v, C);
        qi = exact::ld_local<4>(pi, ai, v, C);
      } else {
        qm = ldg_u4(mine + r * c.slice_cap + v * 16);
        qi = ldg_u4(mine + r * c.slice_cap + (Cv + v) * 16);
      }
      const float cnt = cnts[r];
      const float nf = __int2float_rn(n);
      const float x = __fadd_rn(cnt, nf);
      // ATen writes factor = 1.0 / (n + count), a double division rounded to float.  Its nvcc emits the float reciprocal
      // instead: the double quotient rounded to float is the correctly rounded float quotient (53 >= 2 * 24 + 2 bits).
      const float factor = __frcp_rn(x);
      const float nfac = __fmul_rn(nf, factor);
      const float cfac = __fmul_rn(cnt, factor);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        bnstats::merge(avg[k], var_n[k], bnstats::lane(qm, k), bnstats::lane(qi, k), nf, cnt, factor, nfac, cfac, eps);
      n = __float2int_rz(x);  // index_t n += count: truncation
    }
    const float nf = __int2float_rn(n);
    const float nf1 = __int2float_rn(n - 1);
    float os[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) os[k] = __frcp_rn(__fsqrt_rn(__fadd_rn(__fdiv_rn(var_n[k], nf), eps)));
    exact::st_local<4>(pm, am, v, C, make_uint4(__float_as_uint(avg[0]), __float_as_uint(avg[1]), __float_as_uint(avg[2]),
                                                __float_as_uint(avg[3])));
    exact::st_local<4>(pi, ai, v, C, make_uint4(__float_as_uint(os[0]), __float_as_uint(os[1]), __float_as_uint(os[2]),
                                                __float_as_uint(os[3])));
    // running = (1 - momentum) * running + momentum * x: ATen's SASS fuses the second product
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const unsigned long long i = v * 4 + k;
      if (i < C) {
        if (running_mean != nullptr) running_mean[i] = __fmaf_rn(avg[k], momentum, __fmul_rn(om, running_mean[i]));
        if (running_var != nullptr)
          running_var[i] = __fmaf_rn(__fdiv_rn(var_n[k], nf1), momentum, __fmul_rn(om, running_var[i]));
      }
    }
  }
  if (!solo) op_end(c);
}
