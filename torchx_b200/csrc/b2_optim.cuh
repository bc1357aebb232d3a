// b2_optim.cuh — the optimizer epilogue of the sharded bucket reduce-scatter (b2_reduce_scatter_step): SGD, Adam and
// AdamW applied to this rank's block of the flat parameter buffer as the reduced gradient leaves phase B, instead of
// storing that gradient into a shard for torch's optimizer to read back.
//
// The arithmetic is that of torch's fused optimizers (torch._fused_sgd_ / _fused_adam_ / _fused_adamw_ of torch 2.11,
// fp32 parameters, no grad scale), restated with explicit roundings from their SASS (DESIGN.md 2.4): every hyper-parameter
// reaches ATen as a double and is rounded to fp32 once; all per-element work is fp32.
#pragma once

#include "b2_dev.cuh"

namespace {

constexpr int kOptMaxRuns = B2_OPT_MAX_RUNS;
constexpr int kOptMaxGroups = B2_OPT_MAX_GROUPS;
constexpr int B2_OPT_F_MAXIMIZE = 1;
constexpr int B2_OPT_F_NESTEROV = 2;
constexpr int B2_OPT_F_MOMENTUM = 4;  // SGD with momentum != 0: the group has a momentum buffer
constexpr uint8_t kOptScalar = 0x40;  // in OptDev::group: the unsharded fused Adam steps this parameter on its scalar path

// One parameter group's hyper-parameters as the kernels use them (fp32, rounded from the doubles on the host exactly as
// ATen's launch rounds them).  SGD: a = momentum, b = 1 - dampening (fp32 subtraction, as the fused kernel does it),
// lr_wd unused.  Adam / AdamW: a = beta1, b = beta2, lr_wd = lr * weight_decay (fp32 product: AdamW's decay factor).
struct OptGroupDev {
  float lr, wd, a, b, eps, lr_wd;
  int flags;  // B2_OPT_F_* above
};

// What the epilogue needs next to the gradient: where this rank's block lives, and which group / step count each element
// of the block belongs to.  Run k covers block elements [begin[k], begin[k+1]); group[k] == B2_OPT_NO_GROUP leaves its
// elements untouched (the pad).  Travels by value in the kernel parameters, like Src.
struct OptDev {
  int kind;
  int nrun;
  float* param;  // element 0 of this rank's block
  float* s0;     // momentum_buffer / exp_avg, `block` elements
  float* s1;     // exp_avg_sq
  unsigned long long off;  // block element of this launch's element 0 (a block larger than a stage region is cut up)
  uint32_t begin[kOptMaxRuns + 1];
  uint8_t group[kOptMaxRuns];  // group index, | kOptScalar when the run's parameter takes ATen's scalar path
  uint16_t pidx[kOptMaxRuns];  // element index within its parameter of the run's first element, modulo 65536
  float step[kOptMaxRuns];  // Adam: the step count this update uses (after the increment); SGD: != 0 on the first step
  OptGroupDev g[kOptMaxGroups];
};

}  // namespace

namespace dev {

// The group index of run k (B2_OPT_NO_GROUP for the pad).
__device__ __forceinline__ int opt_group(const OptDev& o, int k) {
  const int g = o.group[k];
  return g == B2_OPT_NO_GROUP ? g : (g & ~kOptScalar);
}

// Per run, once per CTA (Adam / AdamW): ATen's bias corrections and step size.
//   bc1 = 1 - powf(beta1, step);  bc2_sqrt = sqrtf(1 - powf(beta2, step));  step_size = lr / bc1
struct OptCta {
  float step_size[kOptMaxRuns];
  float bc2_sqrt[kOptMaxRuns];
};

__device__ __forceinline__ void opt_cta_init(const OptDev& o, OptCta& t) {
  if (o.kind == B2_OPT_SGD) return;
  for (int k = threadIdx.x; k < o.nrun; k += blockDim.x) {
    const int gi = opt_group(o, k);
    if (gi == B2_OPT_NO_GROUP) continue;
    const OptGroupDev& g = o.g[gi];
    const float bc1 = __fsub_rn(1.f, powf(g.a, o.step[k]));
    const float bc2 = __fsub_rn(1.f, powf(g.b, o.step[k]));
    t.step_size[k] = __fdiv_rn(g.lr, bc1);
    t.bc2_sqrt[k] = __fsqrt_rn(bc2);
  }
}

// Whether ATen's fused Adam rounds `param * weight_decay` before adding it to a non-maximized gradient, for block element
// `e` of run k.  Its unrolled loop over the kILP = 4 elements a thread holds hoists that product out of the maximize branch
// for the first of the four only; the other three are contracted into an FFMA.  Which of the four an element is depends on
// its index j within its parameter: j % 4 on the vectorised path, (j % 65536) % 2048 / 512 on the scalar path (a numel
// that is not a multiple of 4; the 65536-element chunks of 512 threads).
__device__ __forceinline__ bool adam_decay_rounded(const OptDev& o, int k, unsigned long long e) {
  const uint32_t j = (static_cast<uint32_t>(o.pidx[k]) + static_cast<uint32_t>(e - o.begin[k])) & 0xffffu;
  return (o.group[k] & kOptScalar) ? ((j & 2047u) >> 9) == 0 : (j & 3u) == 0;
}

// One element, block element e of run k.  p, m, v: parameter and state in / out; grad: the reduced gradient.
__device__ __forceinline__ void opt_elem(const OptDev& o, const OptCta& t, int k, unsigned long long e, float& p, float grad,
                                         float& m, float& v) {
  const OptGroupDev& g = o.g[opt_group(o, k)];
  if (g.flags & B2_OPT_F_MAXIMIZE) grad = -grad;
  if (o.kind == B2_OPT_SGD) {
    if (g.wd != 0.f) grad = __fmaf_rn(p, g.wd, grad);            // g += weight_decay * p
    if (g.flags & B2_OPT_F_MOMENTUM) {
      // momentum * buf + (1 - dampening) * g: nvcc contracts the other product of ATen's expression when g was negated
      // and not decayed (maximize, weight_decay == 0), in the vectorised path that aligned parameters take
      const bool neg_only = (g.flags & B2_OPT_F_MAXIMIZE) && g.wd == 0.f;
      const float buf = o.step[k] != 0.f ? grad                   // first step: buf = g
                        : neg_only ? __fmaf_rn(m, g.a, __fmul_rn(grad, g.b))
                                   : __fmaf_rn(g.b, grad, __fmul_rn(m, g.a));
      m = buf;
      grad = (g.flags & B2_OPT_F_NESTEROV) ? __fmaf_rn(buf, g.a, grad) : buf;         // g + momentum * buf
    }
    p = __fmaf_rn(grad, -g.lr, p);                                // p -= lr * g
    return;
  }
  if (g.wd != 0.f) {
    if (o.kind == B2_OPT_ADAM) {  // g += p * weight_decay
      if ((g.flags & B2_OPT_F_MAXIMIZE) || adam_decay_rounded(o, k, e)) grad = __fadd_rn(grad, __fmul_rn(p, g.wd));
      else grad = __fmaf_rn(p, g.wd, grad);
    } else p = __fmaf_rn(p, -g.lr_wd, p);                           // AdamW: p -= lr * weight_decay * p
  }
  m = __fmaf_rn(m, g.a, __fmaf_rn(grad, -g.a, grad));             // fma(beta1, m, fma(-beta1, g, g))
  const float gg = __fmul_rn(grad, grad);
  v = __fmaf_rn(v, g.b, __fmaf_rn(gg, -g.b, gg));                 // fma(beta2, v, fma(-beta2, g*g, g*g))
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), t.bc2_sqrt[k]), g.eps);
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(t.step_size[k], m), denom));  // p -= step_size * m / denom
}

// The run a thread looked at last: successive vecs of one thread usually stay inside one parameter.
struct RunHint {
  int k = 0;
  unsigned long long lo = 1, hi = 0;  // empty: the first lookup searches
};

__device__ __forceinline__ int opt_run(const OptDev& o, RunHint& h, unsigned long long e) {
  if (e < h.lo || e >= h.hi) {
    int lo = 0, hi = o.nrun;  // begin[lo] <= e < begin[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (e >= o.begin[mid]) lo = mid;
      else hi = mid;
    }
    h.k = lo;
    h.lo = o.begin[lo];
    h.hi = o.begin[lo + 1];
  }
  return h.k;
}

// The epilogue on one vec: launch elements [e, e + 8) of n, reduced gradient `gr` (fp32 values).  Loads this rank's
// parameter and state slices at the same block offset, steps the elements that belong to a group, stores them back.
__device__ __forceinline__ void opt_step_vec(const OptDev& o, const OptCta& t, RunHint& h, unsigned long long e, unsigned long long n,
                                             const F8& gr) {
  const unsigned long long b = o.off + e;  // block coordinates
  const int k0 = opt_run(o, h, b);
  const bool adam = o.kind != B2_OPT_SGD;
  const bool whole = e + 8 <= n && b + 8 <= h.hi && o.group[k0] != B2_OPT_NO_GROUP;
  const int g0 = opt_group(o, k0);
  float* pp = o.param + b;
  float* p0 = o.s0 + b;
  float* p1 = o.s1 + b;
  const bool vec = whole && ((reinterpret_cast<uintptr_t>(pp) | reinterpret_cast<uintptr_t>(p0) |
                              (adam ? reinterpret_cast<uintptr_t>(p1) : 0)) & 31u) == 0;
  if (vec) {  // one run, one group, 32 B-aligned: vector accesses
    const bool mom = adam || (o.g[g0].flags & B2_OPT_F_MOMENTUM);
    F8 p = ldg_f8(pp), m, v;
    if (mom) m = ldg_f8(p0);
    if (adam) v = ldg_f8(p1);
#pragma unroll
    for (int i = 0; i < 8; ++i) opt_elem(o, t, k0, b + i, p.v[i], gr.v[i], m.v[i], v.v[i]);
    stg_f8(pp, p);
    if (mom) stg_f8(p0, m);
    if (adam) stg_f8(p1, v);
    return;
  }
  int k = k0;
  unsigned long long hi = h.hi;
#pragma unroll
  for (int i = 0; i < 8; ++i) {  // straddles runs (a parameter or group boundary, the pad), misaligned, or the ragged tail
    if (e + i >= n) continue;
    while (b + i >= hi) hi = o.begin[++k + 1];
    const int gi = opt_group(o, k);
    if (gi == B2_OPT_NO_GROUP) continue;
    const bool mom = adam || (o.g[gi].flags & B2_OPT_F_MOMENTUM);
    float p = pp[i], m = mom ? p0[i] : 0.f, v = adam ? p1[i] : 0.f;
    opt_elem(o, t, k, b + i, p, gr.v[i], m, v);
    pp[i] = p;
    if (mom) p0[i] = m;
    if (adam) p1[i] = v;
  }
}

}  // namespace dev
