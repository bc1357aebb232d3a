// b2_bn.cuh — the elementwise passes of training-mode BatchNorm2d on channels-last bf16 activations
// (b2_bn_forward_elemt / b2_bn_backward_elemt).
//
// The data is the row-major [M, C] view of an NHWC-contiguous tensor (M = N*H*W).  Each thread owns one 16-byte vec of
// 8 channels and walks rows; a CTA covers a tile of `cw` vecs x `rows` rows per trip and U trips' loads are issued
// before any is used.
//   k_bn2d_norm       read x, write y       invstd = rsqrt(var + eps), y = w * (x - mean) * invstd + b
//   k_bn2d_bwd_elemt  read x, dy, write dx  dx = (dy - sum_dy/M - (x - mean) * invstd^2 * sum_dy_xmu/M) * invstd * w
// Their inputs are ATen's own reductions (batch_norm_update_stats' mean / var, batch_norm_backward_reduce's sums) and their
// arithmetic is that of ATen's batch_norm_update_stats_and_invert, batch_norm_transform_input_channels_last_kernel and
// batch_norm_backward_elemt_channels_last_kernel, expression for expression: y, invstd and dx are ATen's bits.
// Both passes walk their row blocks last one first: the reduction before them streams the rows upwards, so a layer that
// fits in L2 starts on the rows it read last.
#pragma once

#include <cuda_bf16.h>

#include "b2_dev.cuh"

namespace bn {

// 3 CTAs of 256 threads per SM: up to 80 registers, which the elementwise kernels need for 32 per-channel constants and
// their loads in flight without spilling; 768 threads x 4 vecs keep 48 KiB of loads in flight per SM.
constexpr int kBnThreads = 256;
constexpr int kBnCtasPerSm = 3;

// Launch geometry of one [M, C] layer.
struct Plan {
  int cw;    // vecs (8 channels each) per CTA tile: min(C / 8, kBnThreads)
  int rows;  // rows per trip: kBnThreads / cw
  int gx;    // column tiles
  int gy;    // CTAs along M
};

__host__ __device__ inline Plan plan(unsigned long long M, unsigned long long C, int sms, int unroll) {
  Plan p;
  const unsigned long long cv = C / 8;
  p.cw = static_cast<int>(cv < kBnThreads ? cv : kBnThreads);
  p.rows = kBnThreads / p.cw;
  p.gx = static_cast<int>((cv + p.cw - 1) / p.cw);
  const unsigned long long per = static_cast<unsigned long long>(p.rows) * unroll;
  unsigned long long gy = (M + per - 1) / per;
  unsigned long long cap = static_cast<unsigned long long>(sms) * kBnCtasPerSm / p.gx;
  if (cap < 1) cap = 1;
  if (gy > cap) gy = cap;
  p.gy = static_cast<int>(gy);
  return p;
}

// 8 bf16 lanes of a 16-byte vec <-> fp32
__device__ __forceinline__ void unpack(const uint4& q, float (&f)[8]) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f[2 * k] = __uint_as_float(w[k] << 16);
    f[2 * k + 1] = __uint_as_float(w[k] & 0xFFFF0000u);
  }
}

__device__ __forceinline__ uint4 pack(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
    memcpy(&w[k], &h, 4);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ uint4 ld_vec(const uint16_t* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// The thread's vec column and row within the tile; `on` = it has a column (cw * rows can fall short of the CTA, and the
// last column tile can be partial).
struct Lane {
  unsigned long long col;  // first channel of this thread's vec
  int r;
  bool on;
};

__device__ __forceinline__ Lane lane(const Plan& p, unsigned long long C) {
  Lane l;
  const int t = threadIdx.x;
  l.r = t / p.cw;
  l.col = (static_cast<unsigned long long>(blockIdx.x) * p.cw + t % p.cw) * 8;
  l.on = l.r < p.rows && l.col < C;
  return l;
}

}  // namespace bn

// ---- forward normalise --------------------------------------------------------------------------------------------------
// invstd = rsqrt(var + eps) (ATen's batch_norm_update_stats_and_invert), written to save_invstd by the first CTA row, and
// y = w * (x - mean) * invstd + b in batch_norm_transform_input_channels_last_kernel's order.
template <int U>
__global__ void __launch_bounds__(bn::kBnThreads, bn::kBnCtasPerSm)
    k_bn2d_norm(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, unsigned long long M, unsigned long long C, bn::Plan p,
                const float* __restrict__ mean, const float* __restrict__ var, float eps, float* __restrict__ save_invstd,
                const float* __restrict__ weight, const float* __restrict__ bias) {
  using namespace bn;
  const Lane l = lane(p, C);
  if (!l.on) return;
  float m[8], is[8], w[8], b[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    m[k] = mean[l.col + k];
    is[k] = rsqrtf(var[l.col + k] + eps);
    w[k] = weight[l.col + k];
    b[k] = bias[l.col + k];
  }
  if (blockIdx.y == 0 && l.r == 0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) save_invstd[l.col + k] = is[k];
  }
  const unsigned long long step = static_cast<unsigned long long>(p.rows) * U;
  const unsigned long long stride = step * p.gy;
  const unsigned long long first = blockIdx.y * step;
  if (first >= M) return;
  // last row block first
  for (long long base = static_cast<long long>(first + (M - 1 - first) / stride * stride); base >= 0; base -= stride) {
    uint4 q[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long row = base + u * p.rows + l.r;
      q[u] = row < M ? ld_vec(x + row * C + l.col) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long row = base + u * p.rows + l.r;
      if (row < M) {
        float f[8];
        unpack(q[u], f);
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = w[k] * (f[k] - m[k]) * is[k] + b[k];
        *reinterpret_cast<uint4*>(y + row * C + l.col) = pack(f);
      }
    }
  }
}

// ---- backward elementwise ------------------------------------------------------------------------------------------------
// ATen's per-channel constants (batch_norm_backward_elemt): m_dy = sum_dy / M, f1 = invstd^2 * sum_dy_xmu / M, f2 = w * invstd.
template <int U>
__global__ void __launch_bounds__(bn::kBnThreads, bn::kBnCtasPerSm)
    k_bn2d_bwd_elemt(const uint16_t* __restrict__ dy, const uint16_t* __restrict__ x, uint16_t* __restrict__ dx, unsigned long long M,
                     unsigned long long C, bn::Plan p, const float* __restrict__ mean, const float* __restrict__ invstd,
                     const float* __restrict__ weight, const float* __restrict__ sum_dy, const float* __restrict__ sum_dy_xmu,
                     float norm_fct) {
  using namespace bn;
  const Lane l = lane(p, C);
  if (!l.on) return;
  float m[8], mdy[8], f1[8], f2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const unsigned long long c = l.col + k;
    m[k] = mean[c];
    mdy[k] = sum_dy[c] * norm_fct;
    const float is = invstd[c];
    f2[k] = weight[c] * is;
    f1[k] = is * is * sum_dy_xmu[c] * norm_fct;
  }
  const unsigned long long step = static_cast<unsigned long long>(p.rows) * U;
  const unsigned long long stride = step * p.gy;
  const unsigned long long first = blockIdx.y * step;
  if (first >= M) return;
  for (long long base = static_cast<long long>(first + (M - 1 - first) / stride * stride); base >= 0; base -= stride) {
    uint4 qd[U], qx[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long row = base + u * p.rows + l.r;
      qd[u] = row < M ? ld_vec(dy + row * C + l.col) : make_uint4(0, 0, 0, 0);
      qx[u] = row < M ? ld_vec(x + row * C + l.col) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long row = base + u * p.rows + l.r;
      if (row < M) {
        float fd[8], fx[8];
        unpack(qd[u], fd);
        unpack(qx[u], fx);
#pragma unroll
        for (int k = 0; k < 8; ++k) fd[k] = (fd[k] - mdy[k] - (fx[k] - m[k]) * f1[k]) * f2[k];
        *reinterpret_cast<uint4*>(dx + row * C + l.col) = pack(fd);
      }
    }
  }
}
