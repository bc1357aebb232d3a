// b2_bn.cuh — training-mode BatchNorm2d on channels-last bf16 activations: the two reductions (b2_bn_stats /
// b2_bn_backward_reduce) and the two elementwise passes (b2_bn_forward_elemt / b2_bn_backward_elemt).
//
// The data is the row-major [M, C] view of an NHWC-contiguous tensor (M = N*H*W).  Each thread owns one 16-byte vec of
// 8 channels and walks rows.
//   k_bn2d_stats       read x                mean, var = m2n / M, running statistics (ATen's Welford tree, below)
//   k_bn2d_bwd_reduce  read x, dy            sum_dy, sum_dy_xmu, grad_weight = sum_dy_xmu * invstd, grad_bias = sum_dy
//   k_bn2d_norm        read x, write y       invstd = rsqrt(var + eps), y = w * (x - mean) * invstd + b
//   k_bn2d_bwd_elemt   read x, dy, write dx  dx = (dy - sum_dy/M - (x - mean) * invstd^2 * sum_dy_xmu/M) * invstd * w
// SyncBatchNorm runs the same kernels with runtime arguments for its differences (torch.batch_norm_stats,
// batch_norm_elemt and the count form of batch_norm_backward_elemt): the statistics write invstd (ATen's InvStd) instead
// of var, the normalise takes the merged invstd as given, and dx's 1/M comes from the ranks' counts.
// ResNet blocks fold their ReLU and residual add into two of them (b2_bn_forward_relu / b2_bn_backward_reduce_relu):
//   k_bn2d_norm        + read residual       z = relu(bf16(bf16(y) + residual)): ATen's bf16 add_, then relu_
//   k_bn2d_bwd_reduce  read dz, z, x, write dy  dy = threshold_backward(dz, z, 0), then the sums over dy
// The arithmetic is that of ATen's batch_norm_collect_statistics_channels_last_kernel, batch_norm_update_stats(_and_invert),
// batch_norm_backward_reduce_channels_last_kernel, batch_norm_transform_input_channels_last_kernel and
// batch_norm_backward_elemt_channels_last_kernel, expression for expression and, for the reductions, in ATen's order:
// every output is ATen's bits (DESIGN.md 2.4).
// The reductions walk the rows upwards and the elementwise passes walk their row blocks last one first, so a layer that
// fits in L2 starts on the rows the reduction read last.
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

// A coherent load, for data the kernel may overwrite (the fused reduce's dz, when dy_out is dz)
__device__ __forceinline__ uint4 ld_vec_rw(const uint16_t* p) { return *reinterpret_cast<const uint4*>(p); }

__device__ __forceinline__ float round_bf16(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// What the fused forward does to the BatchNorm output y of one element, in the unfused composition's steps: y is stored
// as bf16; the residual add is ATen's bf16 add_ (fp32 opmath, round to nearest even); relu is ATen's relu_, clamp_min(0)
// on the bf16 value, which lets a NaN through.
__device__ __forceinline__ float fuse_out(float y, bool add, float r, bool relu) {
  float v = round_bf16(y);
  if (add) v = round_bf16(__fadd_rn(v, r));
  if (relu && !isnan(v)) v = fmaxf(v, 0.0f);
  return v;
}

// threshold_backward(dz, z, 0) lane by lane on the bf16 words: +0 where z <= 0, dz elsewhere (a NaN z keeps dz).
__device__ __forceinline__ uint4 relu_grad(const uint4& dz, const uint4& z) {
  float fz[8];
  unpack(z, fz);
  uint32_t w[4] = {dz.x, dz.y, dz.z, dz.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t lo = fz[2 * k] <= 0.0f ? 0u : w[k] & 0x0000FFFFu;
    const uint32_t hi = fz[2 * k + 1] <= 0.0f ? 0u : w[k] & 0xFFFF0000u;
    w[k] = lo | hi;
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

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

// ---- ATen's reduction tree ------------------------------------------------------------------------------------------------
// ATen's channels-last reductions launch flexible_launch_configs(M, C, block, grid, coop = true) with 4 parallel loads per
// thread.  A channel's result depends only on block.y and grid.y: thread (ty, by) with slot j runs one sequential chain over
// rows by*block_y + ty + (4i + j)*S, S = block_y*grid_y, i < loops; the 4 slots merge in order, then the block_y threads
// of a CTA pairwise by halving offsets, then (grid_y > 1) the CTA partials in ATen's last-block order.  block.x only decides
// which channels share a CTA.  Every quantity here is a function of the shape alone (no device query), and M*C < 2^31.
constexpr int kAtenMaxBlock = 512;      // MAX_BLOCK_SIZE
constexpr int kAtenTileW = 32;          // OPTIMAL_TILE_W
constexpr int kAtenElemsPerThread = 16; // ELEMENTS_PER_THREAD
constexpr int kAtenMaxHBlock = 128;     // MAX_H_BLOCK
constexpr int kAtenLoads = 4;           // ELEMENTS_PER_ITER, the kernels' PARALLEL_LOADS

struct Tree {
  int block_x, block_y, grid_x, grid_y;  // ATen's launch
  int seq;    // S = block_y * grid_y
  int loops;  // loop_count: rows per chain, the same for every chain
};

inline int last_pow2(unsigned n) {
  n |= n >> 1;
  n |= n >> 2;
  n |= n >> 4;
  n |= n >> 8;
  n |= n >> 16;
  const int p = static_cast<int>(n - (n >> 1));
  return p > 1 ? p : 1;
}

inline Tree tree(int M, int C) {
  Tree t;
  const int lp = last_pow2(static_cast<unsigned>(C));
  t.block_x = lp < kAtenTileW ? lp : kAtenTileW;
  const int by = last_pow2(static_cast<unsigned>((M + kAtenElemsPerThread - 1) / kAtenElemsPerThread));
  t.block_y = by < kAtenMaxBlock / t.block_x ? by : kAtenMaxBlock / t.block_x;
  if (t.block_x * t.block_y != kAtenMaxBlock) t.block_x = lp < kAtenMaxBlock / t.block_y ? lp : kAtenMaxBlock / t.block_y;
  t.grid_x = (C + t.block_x - 1) / t.block_x;
  const int gy = (M + t.block_y * kAtenElemsPerThread - 1) / (t.block_y * kAtenElemsPerThread);
  t.grid_y = gy < kAtenMaxHBlock ? gy : kAtenMaxHBlock;
  if (t.grid_y < 8) t.grid_y = 1;  // coop_flag
  t.seq = t.block_y * t.grid_y;
  t.loops = 1 + (M - 1) / (t.seq * kAtenLoads);
  return t;
}

// Our CTA: `vw` vecs x block_y x the 4 slots, one chain of 8 channels per thread (vec fastest, so a warp reads whole
// rows); one CTA row per ATen CTA row (blockIdx.y = by).  block_y <= 512 / 8, so a CTA has at most 256 threads.  The
// grid_y merge: `mw` vecs x block_y threads per CTA.  reduce_rows and reduce_partials decode these from threadIdx.x.
struct ReduceGrid {
  int vw, block;
  dim3 grid;
  int mw, merge_block, merge_grid;
};

inline ReduceGrid reduce_grid(const Tree& t, int C) {
  const auto vecs = [C](int per) {  // vecs of `per` threads each in one CTA
    const int w = kBnThreads / per > 1 ? kBnThreads / per : 1;
    return w < C / 8 ? w : C / 8;
  };
  ReduceGrid g;
  g.vw = vecs(t.block_y * kAtenLoads);
  g.block = g.vw * t.block_y * kAtenLoads;
  g.grid = dim3((C / 8 + g.vw - 1) / g.vw, t.grid_y);
  g.mw = vecs(t.block_y);
  g.merge_block = g.mw * t.block_y;
  g.merge_grid = (C / 8 + g.mw - 1) / g.mw;
  return g;
}

// Partials of the grid_y merge, float [by][C] mean (sum_dy) and m2n (sum_dy_xmu) and, for the statistics, int [by][C/8]
// counts: ATen's staging, 3 words per (channel, by) there.
inline size_t workspace_bytes(const Tree& t, int C) {
  return t.grid_y > 1 ? static_cast<size_t>(t.grid_y) * (2 * static_cast<size_t>(C) + C / 8) * 4 : 0;
}

// Welford state of one chain over 8 channels (the count is the same for all 8: rows are valid for a whole vec or not at all).
struct Welford {
  static constexpr int kIn = 1;  // inputs: x
  int n;
  float mean[8], m2n[8];
};

// ATen's welford_merge_element, in the two contractions its build uses (sm_90 SASS, DESIGN.md 2.4): merging the 4 slots
// inside a thread fuses mean_new * count_new (FFMA mean_new, cn, mean * c), every other merge fuses mean * count.  A
// zero-count merge is not skipped: (mean * c) * (1 / max(1, c)) can change bits, as in ATen.
template <bool kSlots>
__device__ __forceinline__ void welford_merge(Welford& a, int cn, const float (&mn)[8], const float (&m2)[8]) {
  const int tot = a.n + cn;
  const float factor = __frcp_rn(__int2float_rn(tot > 1 ? tot : 1));
  const float fc = __int2float_rn(a.n), fcn = __int2float_rn(cn);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float d0 = __fsub_rn(a.mean[k], mn[k]);
    const float t = __fmul_rn(fc, __fmul_rn(fcn, __fmul_rn(d0, d0)));
    const float s = kSlots ? __fmaf_rn(mn[k], fcn, __fmul_rn(a.mean[k], fc)) : __fmaf_rn(a.mean[k], fc, __fmul_rn(mn[k], fcn));
    a.mean[k] = __fmul_rn(s, factor);
    a.m2n[k] = __fadd_rn(a.m2n[k], __fmaf_rn(t, factor, m2[k]));
  }
  a.n = tot;
}

// The backward reduce's state of one chain over 8 channels: sum_dy and sum_dy_xmu.  The member order is deliberate: it
// decides how ptxas assigns registers in both reduce kernels.
struct Sums {
  static constexpr int kIn = 2;  // inputs: dy, x
  float xmu[8], dy[8];
};

// Shared-memory slots of a CTA's states: [8][256] means and m2ns (sum_dy / sum_dy_xmu), [256] counts.
struct Smem {
  float a[8][kBnThreads];
  float b[8][kBnThreads];
  int n[kBnThreads];
};

// ---- what the reduction skeletons do with each state ---------------------------------------------------------------------
// zero: the state a chain starts from.  begin: the chain's per-channel constants m (the backward's mean), loaded only by
// threads with a vec.  update: one row of the inputs; `in` = the row is below M.

__device__ __forceinline__ void zero(Welford& w) {
  w.n = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) w.mean[k] = w.m2n[k] = 0.0f;
}

__device__ __forceinline__ void zero(Sums& s) {
#pragma unroll
  for (int k = 0; k < 8; ++k) s.dy[k] = s.xmu[k] = 0.0f;
}

__device__ __forceinline__ void begin(const Welford&, float (&)[8], const float*, unsigned long long) {}

__device__ __forceinline__ void begin(const Sums&, float (&m)[8], const float* mean, unsigned long long col) {
#pragma unroll
  for (int k = 0; k < 8; ++k) m[k] = mean[col + k];
}

// ATen's Welford update in ATen's contraction (delta0 = x - mean; mean = FFMA delta0, 1/count, mean; delta1 = x - mean;
// m2n = FFMA delta0*delta1, is_valid, m2n), one IEEE reciprocal of the count per row for all 8 channels.  A slot past M
// still runs the update with x = 0, 1/count = 0, is_valid = 0, as ATen's does: that is not a no-op once the mean is inf
// or NaN.
__device__ __forceinline__ void update(Welford& w, const float (&)[8], bool in, const float (&f)[1][8]) {
  float inv = 0.0f, valid = 0.0f;
  if (in) {
    ++w.n;
    inv = __frcp_rn(__int2float_rn(w.n));
    valid = 1.0f;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float d0 = __fsub_rn(f[0][k], w.mean[k]);
    w.mean[k] = __fmaf_rn(d0, inv, w.mean[k]);
    const float d1 = __fsub_rn(f[0][k], w.mean[k]);
    w.m2n[k] = __fmaf_rn(__fmul_rn(d0, d1), valid, w.m2n[k]);
  }
}

// sum_dy += dy (FADD), sum_dy_xmu = FFMA (x - mean), dy, sum_dy_xmu; a slot past M adds dy = 0 and 0 * (0 - mean).
__device__ __forceinline__ void update(Sums& s, const float (&m)[8], bool, const float (&f)[2][8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    s.dy[k] = __fadd_rn(s.dy[k], f[0][k]);
    s.xmu[k] = __fmaf_rn(__fsub_rn(f[1][k], m[k]), f[0][k], s.xmu[k]);
  }
}

__device__ __forceinline__ void put(Smem& s, int slot, const Welford& w) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    s.a[k][slot] = w.mean[k];
    s.b[k][slot] = w.m2n[k];
  }
  s.n[slot] = w.n;
}

template <bool kSlots>
__device__ __forceinline__ void merge_from(Welford& w, const Smem& s, int slot) {
  float mn[8], m2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    mn[k] = s.a[k][slot];
    m2[k] = s.b[k][slot];
  }
  welford_merge<kSlots>(w, s.n[slot], mn, m2);
}

__device__ __forceinline__ void put(Smem& s, int slot, const Sums& w) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    s.a[k][slot] = w.dy[k];
    s.b[k][slot] = w.xmu[k];
  }
}

// Every merge of the sums is one FADD, the slots' as the tree's.
template <bool kSlots>
__device__ __forceinline__ void merge_from(Sums& w, const Smem& s, int slot) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    w.dy[k] = __fadd_rn(w.dy[k], s.a[k][slot]);
    w.xmu[k] = __fadd_rn(w.xmu[k], s.b[k][slot]);
  }
}

// CTA row blockIdx.y's partial into the workspace.
__device__ __forceinline__ void store_partial(float* ws, int grid_y, int C, unsigned long long col, int vec, const Welford& w) {
  const size_t base = static_cast<size_t>(blockIdx.y) * C + col;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    ws[base + k] = w.mean[k];
    ws[static_cast<size_t>(grid_y) * C + base + k] = w.m2n[k];
  }
  reinterpret_cast<int*>(ws + 2 * static_cast<size_t>(grid_y) * C)[static_cast<size_t>(blockIdx.y) * (C / 8) + vec] = w.n;
}

__device__ __forceinline__ void store_partial(float* ws, int grid_y, int C, unsigned long long col, int, const Sums& s) {
  const size_t base = static_cast<size_t>(blockIdx.y) * C + col;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    ws[base + k] = s.dy[k];
    ws[static_cast<size_t>(grid_y) * C + base + k] = s.xmu[k];
  }
}

// Merges CTA row y's partial, whose two float halves the skeleton has read into a and b (cnt: the statistics' counts).
__device__ __forceinline__ void fold_partial(Welford& w, const float (&a)[8], const float (&b)[8], const int* cnt, int C, int vec, int y) {
  welford_merge<false>(w, cnt[static_cast<size_t>(y) * (C / 8) + vec], a, b);
}

__device__ __forceinline__ void fold_partial(Sums& s, const float (&a)[8], const float (&b)[8], const int*, int, int, int) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    s.dy[k] = __fadd_rn(s.dy[k], a[k]);
    s.xmu[k] = __fadd_rn(s.xmu[k], b[k]);
  }
}

// ATen's welford_merge_block_vertical / merge_block_vertical_backward over ty (slot = v + vw * ty): ty < off takes ty + off
// for off = block_y/2 .. 1.  Every thread of the CTA calls it; `live` threads hold a state.
template <class S>
__device__ __forceinline__ void vertical(Smem& sm, S& s, int v, int vw, int ty, int block_y, bool live) {
  for (int off = block_y / 2; off > 0; off >>= 1) {
    __syncthreads();
    if (live && ty < off) {
      merge_from<false>(s, sm, v + vw * (ty + off));
      put(sm, v + vw * ty, s);
    }
  }
}

// ATen's InvStd transform of torch.batch_norm_stats: its eps parameter is a double, so var + eps, the square root and the
// reciprocal are IEEE double operations (sm_90 SASS: F2F.F64.F32 of var and of the float eps, DADD, MUFU.RSQ64H + Newton,
// MUFU.RCP64H + Newton), rounded to float once; 0 where var and eps are both zero.
__device__ __forceinline__ float inv_std(float var, float eps) {
  if (var == 0.0f && eps == 0.0f) return 0.0f;
  return __double2float_rn(__drcp_rn(__dsqrt_rn(__dadd_rn(static_cast<double>(var), static_cast<double>(eps)))));
}

// The end of ATen's statistics kernel and of batch_norm_update_stats_and_invert's running-statistics lambda (fp32:
// 1 - momentum by FADD, FMUL (1 - momentum) * running, FFMA x, momentum, that; bessel = M / (M - 1) in double rounded to
// float at the launch).  With `invstd` the second output is inv_std(var, eps) (torch.batch_norm_stats, which updates no
// running statistics: the host passes none).
__device__ __forceinline__ void stats_out(const Welford& w, unsigned long long col, float* __restrict__ mean, float* __restrict__ var,
                                          float* __restrict__ running_mean, float* __restrict__ running_var, float momentum, float bessel,
                                          bool invstd, float eps) {
  const float omm = __fsub_rn(1.0f, momentum);
  const float fn = __int2float_rn(w.n);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float v = __fdiv_rn(w.m2n[k], fn);
    mean[col + k] = w.mean[k];
    var[col + k] = invstd ? inv_std(v, eps) : v;
    if (running_mean != nullptr) {
      running_mean[col + k] = __fmaf_rn(w.mean[k], momentum, __fmul_rn(omm, running_mean[col + k]));
      running_var[col + k] = __fmaf_rn(__fmul_rn(v, bessel), momentum, __fmul_rn(omm, running_var[col + k]));
    }
  }
}

// The end of ATen's backward reduce: grad_weight = sum_dy_xmu * invstd (FMUL), grad_bias = sum_dy.
__device__ __forceinline__ void reduce_out(const Sums& s, unsigned long long col, const float* __restrict__ invstd, float* __restrict__ sum_dy,
                                           float* __restrict__ sum_dy_xmu, float* __restrict__ grad_weight, float* __restrict__ grad_bias) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sum_dy[col + k] = s.dy[k];
    sum_dy_xmu[col + k] = s.xmu[k];
    grad_weight[col + k] = __fmul_rn(s.xmu[k], invstd[col + k]);
    grad_bias[col + k] = s.dy[k];
  }
}

// ---- the skeletons ------------------------------------------------------------------------------------------------------
// The elementwise passes: each CTA row walks its row blocks of p.rows * U rows, last one first, with U rows' loads of
// every input issued before the first is used.  f(in, out) maps one row's 8 channels of the kIn inputs to the output's.
template <int U, int kIn, class F>
__device__ __forceinline__ void elemt_rows(const Lane& l, const Plan& p, unsigned long long M, unsigned long long C,
                                           const uint16_t* __restrict__ in0, const uint16_t* __restrict__ in1, uint16_t* __restrict__ out,
                                           F&& f) {
  const unsigned long long step = static_cast<unsigned long long>(p.rows) * U;
  const unsigned long long stride = step * p.gy;
  const unsigned long long first = blockIdx.y * step;
  if (first >= M) return;
  for (long long base = static_cast<long long>(first + (M - 1 - first) / stride * stride); base >= 0; base -= stride) {
    uint4 q[U][kIn];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long row = base + u * p.rows + l.r;
      q[u][0] = row < M ? ld_vec(in0 + row * C + l.col) : make_uint4(0, 0, 0, 0);
      if constexpr (kIn == 2) q[u][1] = row < M ? ld_vec(in1 + row * C + l.col) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long row = base + u * p.rows + l.r;
      if (row < M) {
        float fi[kIn][8], fo[8];
#pragma unroll
        for (int i = 0; i < kIn; ++i) unpack(q[u][i], fi[i]);
        f(fi, fo);
        *reinterpret_cast<uint4*>(out + row * C + l.col) = pack(fo);
      }
    }
  }
}

// One thread's chain of state S over the S::kIn inputs (in0, in1) from `row`, with U rows' loads issued before the first is
// used.  kMask (the backward reduce only): in0 is dz, and each row's dy = relu_grad(dz, z) is written to dy_out and summed;
// dy_out may be dz itself (each row is read, then written, by one thread).
template <int U, bool kMask, class S>
__device__ __forceinline__ void chain(S& s, const float (&m)[8], const uint16_t* in0, const uint16_t* in1, const uint16_t* z,
                                      uint16_t* dy_out, int M, int C, const Tree& t, int row, unsigned long long col) {
  constexpr int kLoads = S::kIn + (kMask ? 1 : 0);
  const int stride = kAtenLoads * t.seq;
  for (int i = 0; i < t.loops; i += U) {
    uint4 q[U][kLoads];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = row + u * stride;
      const bool ld = i + u < t.loops && r < M;
      const uint16_t* p0 = in0 + static_cast<unsigned long long>(r) * C + col;
      q[u][0] = ld ? (kMask ? ld_vec_rw(p0) : ld_vec(p0)) : make_uint4(0, 0, 0, 0);
      if constexpr (S::kIn == 2) q[u][1] = ld ? ld_vec(in1 + static_cast<unsigned long long>(r) * C + col) : make_uint4(0, 0, 0, 0);
      if constexpr (kMask) q[u][2] = ld ? ld_vec(z + static_cast<unsigned long long>(r) * C + col) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (i + u < t.loops) {
        const int r = row + u * stride;
        if constexpr (kMask) {
          q[u][0] = relu_grad(q[u][0], q[u][2]);
          if (r < M) *reinterpret_cast<uint4*>(dy_out + static_cast<unsigned long long>(r) * C + col) = q[u][0];
        }
        float f[S::kIn][8];
#pragma unroll
        for (int n = 0; n < S::kIn; ++n) unpack(q[u][n], f[n]);
        update(s, m, r < M, f);
      }
    }
    row += U * stride;
  }
}

// The reductions: thread (vec, ty, j) of ATen CTA row by = blockIdx.y runs its chain; then the slot merge and the
// vertical merge through shared memory.  With grid_y == 1 the CTA hands each vec's state to out(state, col), otherwise it
// writes its partial, which reduce_partials folds.  `mean` feeds begin (the backward's; null for the statistics).  A
// non-null z (the backward reduce's) masks in0 = dz by relu_grad into dy_out.
template <int U, class S, class Out>
__device__ __forceinline__ void reduce_rows(const uint16_t* in0, const uint16_t* in1, int M, int C, const Tree& t, int vw, const float* mean,
                                            float* ws, Out&& out, const uint16_t* z = nullptr, uint16_t* dy_out = nullptr) {
  __shared__ Smem sm;
  const int tid = threadIdx.x;
  const int v = tid % vw, ty = (tid / vw) % t.block_y, j = tid / (vw * t.block_y);
  const int vec = blockIdx.x * vw + v;
  const bool on = vec < C / 8;
  const unsigned long long col = static_cast<unsigned long long>(vec) * 8;
  S s;
  zero(s);
  float m[8];
  if (on) {
    begin(s, m, mean, col);
    const int row = blockIdx.y * t.block_y + ty + j * t.seq;
    // the relu-masked chain has a third input: one row in flight keeps its loads in the registers of the plain chain's
    if constexpr (S::kIn == 2) {
      if (z != nullptr) {
        chain<(U > 1 ? U / 2 : 1), true>(s, m, in0, in1, z, dy_out, M, C, t, row, col);
      } else {
        chain<U, false>(s, m, in0, in1, nullptr, nullptr, M, C, t, row, col);
      }
    } else {
      chain<U, false>(s, m, in0, in1, nullptr, nullptr, M, C, t, row, col);
    }
  }
  put(sm, v + vw * (ty + t.block_y * j), s);
  __syncthreads();
  const bool lead = on && j == 0;
  if (lead) {
#pragma unroll
    for (int jj = 1; jj < kAtenLoads; ++jj) merge_from<true>(s, sm, v + vw * (ty + t.block_y * jj));
    put(sm, v + vw * ty, s);
  }
  vertical(sm, s, v, vw, ty, t.block_y, lead);
  if (!lead || ty != 0) return;
  if (t.grid_y == 1) {
    out(s, col);
    return;
  }
  store_partial(ws, t.grid_y, C, col, vec, s);
}

// ATen's last block: thread ty folds partials y = ty, ty + block_y, ... into a zero state, then the vertical merge, and
// ty = 0 hands each vec's state to out(state, col).
template <class S, class Out>
__device__ __forceinline__ void reduce_partials(int C, const Tree& t, int vw, const float* ws, Out&& out) {
  __shared__ Smem sm;
  const int tid = threadIdx.x;
  const int v = tid % vw, ty = tid / vw;
  const int vec = blockIdx.x * vw + v;
  const bool on = vec < C / 8;
  const unsigned long long col = static_cast<unsigned long long>(vec) * 8;
  const int* cnt = reinterpret_cast<const int*>(ws + 2 * static_cast<size_t>(t.grid_y) * C);
  S s;
  zero(s);
  if (on) {
    for (int y = ty; y < t.grid_y; y += t.block_y) {
      const size_t base = static_cast<size_t>(y) * C + col;
      float a[8], b[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        a[k] = ws[base + k];
        b[k] = ws[static_cast<size_t>(t.grid_y) * C + base + k];
      }
      fold_partial(s, a, b, cnt, C, vec, y);
    }
    put(sm, v + vw * ty, s);
  }
  vertical(sm, s, v, vw, ty, t.block_y, on);
  if (on && ty == 0) out(s, col);
}

}  // namespace bn

// ---- forward normalise --------------------------------------------------------------------------------------------------
// invstd = rsqrt(var + eps) (ATen's batch_norm_update_stats_and_invert), written to save_invstd by the first CTA row, and
// y = w * (x - mean) * invstd + b in batch_norm_transform_input_channels_last_kernel's order.  A null save_invstd means
// var already holds invstd (SyncBatchNorm's merged statistics, which torch.batch_norm_elemt reads as given).  With a residual or relu,
// y goes through fuse_out.  A residual is a second input: its rows go U / 2 at a time, so that the x and residual loads in
// flight fit the registers of x's alone (the plan is made for that unroll).
template <int U>
__global__ void __launch_bounds__(bn::kBnThreads, bn::kBnCtasPerSm)
    k_bn2d_norm(const uint16_t* __restrict__ x, const uint16_t* __restrict__ residual, uint16_t* __restrict__ y, unsigned long long M,
                unsigned long long C, bn::Plan p, const float* __restrict__ mean, const float* __restrict__ var, float eps,
                float* __restrict__ save_invstd, const float* __restrict__ weight, const float* __restrict__ bias, bool relu) {
  using namespace bn;
  const Lane l = lane(p, C);
  if (!l.on) return;
  float m[8], is[8], w[8], b[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    m[k] = mean[l.col + k];
    is[k] = save_invstd != nullptr ? rsqrtf(var[l.col + k] + eps) : var[l.col + k];
    w[k] = weight[l.col + k];
    b[k] = bias[l.col + k];
  }
  if (save_invstd != nullptr && blockIdx.y == 0 && l.r == 0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) save_invstd[l.col + k] = is[k];
  }
  const auto norm = [&](float v, int k) { return w[k] * (v - m[k]) * is[k] + b[k]; };
  if (residual != nullptr) {
    elemt_rows<(U > 1 ? U / 2 : 1), 2>(l, p, M, C, x, residual, y, [&](const float (&f)[2][8], float (&o)[8]) {
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = fuse_out(norm(f[0][k], k), true, f[1][k], relu);
    });
  } else if (relu) {
    elemt_rows<U, 1>(l, p, M, C, x, nullptr, y, [&](const float (&f)[1][8], float (&o)[8]) {
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = fuse_out(norm(f[0][k], k), false, 0.0f, true);
    });
  } else {
    elemt_rows<U, 1>(l, p, M, C, x, nullptr, y, [&](const float (&f)[1][8], float (&o)[8]) {
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = norm(f[0][k], k);
    });
  }
}

// ---- backward elementwise ------------------------------------------------------------------------------------------------
// ATen's per-channel constants (batch_norm_backward_elemt): m_dy = sum_dy / M, f1 = invstd^2 * sum_dy_xmu / M, f2 = w * invstd,
// and per element dx = ((dy - m_dy) - (x - mean) * f1) * f2.  Its sm_90 SASS, whose roundings are written out here (left to
// nvcc, the contraction follows its register allocation): f1 and f2 by FMULs; FADD x - mean; FFMA -(x - mean), f1, t;
// FMUL f2; and t = FFMA -sum_dy, norm_fct, dy in the scalar form (BatchNorm2d), but FADD dy - m_dy with m_dy = FMUL
// sum_dy * norm_fct in the count form (SyncBatchNorm).  With `counts` (every rank's count as float) 1 / M is that of the
// count form: the int64 sum of the counts as int32 (torch's .to(torch.int32) truncates), converted to float, then the IEEE
// float reciprocal (I2F.S64, MUFU.RCP + Newton); otherwise it is the host's norm_fct.
template <int U>
__global__ void __launch_bounds__(bn::kBnThreads, bn::kBnCtasPerSm)
    k_bn2d_bwd_elemt(const uint16_t* __restrict__ dy, const uint16_t* __restrict__ x, uint16_t* __restrict__ dx, unsigned long long M,
                     unsigned long long C, bn::Plan p, const float* __restrict__ mean, const float* __restrict__ invstd,
                     const float* __restrict__ weight, const float* __restrict__ sum_dy, const float* __restrict__ sum_dy_xmu,
                     float norm_fct, const float* __restrict__ counts, int n_counts) {
  using namespace bn;
  const Lane l = lane(p, C);
  if (!l.on) return;
  if (counts != nullptr) {
    long long total = 0;
    for (int i = 0; i < n_counts; ++i) total += __float2int_rz(counts[i]);
    norm_fct = __frcp_rn(__ll2float_rn(total));
  }
  float m[8], mdy[8], f1[8], f2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const unsigned long long c = l.col + k;
    m[k] = mean[c];
    mdy[k] = counts != nullptr ? __fmul_rn(sum_dy[c], norm_fct) : sum_dy[c];  // the scalar form keeps sum_dy
    const float is = invstd[c];
    f2[k] = __fmul_rn(weight[c], is);
    f1[k] = __fmul_rn(__fmul_rn(__fmul_rn(is, is), sum_dy_xmu[c]), norm_fct);
  }
  if (counts != nullptr) {
    elemt_rows<U, 2>(l, p, M, C, dy, x, dx, [&](const float (&f)[2][8], float (&o)[8]) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        o[k] = __fmul_rn(__fmaf_rn(-__fsub_rn(f[1][k], m[k]), f1[k], __fsub_rn(f[0][k], mdy[k])), f2[k]);
    });
  } else {
    elemt_rows<U, 2>(l, p, M, C, dy, x, dx, [&](const float (&f)[2][8], float (&o)[8]) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        o[k] = __fmul_rn(__fmaf_rn(-__fsub_rn(f[1][k], m[k]), f1[k], __fmaf_rn(-mdy[k], norm_fct, f[0][k])), f2[k]);
    });
  }
}

// ---- forward statistics -------------------------------------------------------------------------------------------------
// ATen's Welford chains; the merge kernel folds the CTA rows' partials in ATen's last-block order and, like the main
// kernel with grid_y == 1, writes mean, var = m2n / M (with `invstd`: inv_std(var, eps)) and the running statistics.
template <int U>
__global__ void __launch_bounds__(bn::kBnThreads)
    k_bn2d_stats(const uint16_t* __restrict__ x, int M, int C, bn::Tree t, int vw, float* __restrict__ mean, float* __restrict__ var,
                 float* __restrict__ running_mean, float* __restrict__ running_var, float momentum, float bessel, bool invstd, float eps,
                 float* __restrict__ ws) {
  using namespace bn;
  reduce_rows<U, Welford>(x, nullptr, M, C, t, vw, nullptr, ws, [&](const Welford& w, unsigned long long col) {
    stats_out(w, col, mean, var, running_mean, running_var, momentum, bessel, invstd, eps);
  });
}

__global__ void __launch_bounds__(bn::kBnThreads)
    k_bn2d_stats_merge(int C, bn::Tree t, int vw, const float* __restrict__ ws, float* __restrict__ mean, float* __restrict__ var,
                       float* __restrict__ running_mean, float* __restrict__ running_var, float momentum, float bessel, bool invstd,
                       float eps) {
  using namespace bn;
  reduce_partials<Welford>(C, t, vw, ws, [&](const Welford& w, unsigned long long col) {
    stats_out(w, col, mean, var, running_mean, running_var, momentum, bessel, invstd, eps);
  });
}

// ---- backward reduce ----------------------------------------------------------------------------------------------------
// The same tree with plain sums.  ATen's kernel returns early from threads with c_offset >= C or m_offset >= M: the first
// only ever holds channels no valid thread reads (the vertical merge pairs threads of one threadIdx.x), and m_offset =
// by*block_y + ty < block_y*grid_y <= M for every geometry flexible_launch_configs makes, so no valid channel is affected.
// With z (the fused forward's output) dy is the gradient dz of z: the kernel sums threshold_backward(dz, z, 0) instead,
// in the same order, and writes it to dy_out (every row, by the thread whose chain holds it); dy_out may be dy.
template <int U>
__global__ void __launch_bounds__(bn::kBnThreads)
    k_bn2d_bwd_reduce(const uint16_t* dy, const uint16_t* __restrict__ z, const uint16_t* __restrict__ x, uint16_t* dy_out, int M, int C,
                      bn::Tree t, int vw, const float* __restrict__ mean, const float* __restrict__ invstd, float* __restrict__ sum_dy, float* __restrict__ sum_dy_xmu,
                      float* __restrict__ grad_weight, float* __restrict__ grad_bias, float* __restrict__ ws) {
  using namespace bn;
  reduce_rows<U, Sums>(
      dy, x, M, C, t, vw, mean, ws,
      [&](const Sums& s, unsigned long long col) { reduce_out(s, col, invstd, sum_dy, sum_dy_xmu, grad_weight, grad_bias); }, z, dy_out);
}

__global__ void __launch_bounds__(bn::kBnThreads)
    k_bn2d_bwd_reduce_merge(int C, bn::Tree t, int vw, const float* __restrict__ ws, const float* __restrict__ invstd,
                            float* __restrict__ sum_dy, float* __restrict__ sum_dy_xmu, float* __restrict__ grad_weight,
                            float* __restrict__ grad_bias) {
  using namespace bn;
  reduce_partials<Sums>(C, t, vw, ws, [&](const Sums& s, unsigned long long col) {
    reduce_out(s, col, invstd, sum_dy, sum_dy_xmu, grad_weight, grad_bias);
  });
}
