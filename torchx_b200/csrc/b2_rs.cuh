// b2_rs.cuh — reduce-scatter (b2_reduce_scatter): rank r ends with block r of the allreduce of the W ranks' inputs, and
// each rank moves only (W-1)/W of its input over the fabric.
//   A  push-scatter : block j of my input -> recv[me] of rank j (raw vecs, or wire(scale * x) for a float sum)
//   B  reduce       : combine recv[0..W-1] of my own stage in rank order, write `out`
// One cta_xbar between them.  Phase B is k_twoshot's phase B (float SUM / AVG) or k_reduce_exact's combine (integer SUM,
// MIN / MAX), so block r is the same bits as the allreduce leaves there.
//
// `in` holds W blocks of `block` elements; a launch covers elements [0, n) of every block (the host cuts a block larger
// than a stage region into several launches along the block axis).  The block boundaries j * block need not fall on a
// vec, so every block has its own alignment flag and the element fallbacks of the local accesses handle the rest.  The
// thread that reads vec v of my own block in phase A is the one that writes vec v of `out` in phase B, so `out` may be my
// block of `in` (the in-place form).  The op counter, stage parity and flag sequence are those of every other collective.
//
// The float kernel also reads its input through a segment table (b2_reduce_scatter_gather: the sharded bucket of the
// mini-DDP, zero-copy as b2_allreduce_gather).  `src.nseg == 0` is the flat `in` above; otherwise element i of block j of
// this launch is bucket element j * block + src.off + i, and `in` is not read.
#pragma once

#include "b2_dev.cuh"
#include "b2_exact.cuh"
#include "b2_optim.cuh"

// Phase A of the float kernels: block j of my input -> recv[me] of rank j, as wire(scale * x).
template <int MODE, int W>
__device__ __forceinline__ void rs_scatter(const CommDev& c, const Src& src, const void* in, unsigned long long n,
                                           unsigned long long block, float scale, unsigned long long stage) {
  using namespace dev;
  using Elem = typename ModeTraits<MODE>::Elem;
  constexpr int WVB = Wire<MODE>::kBytes;
  constexpr int U = vecs_per_trip(W);
  const unsigned long long V = (n + 7) / 8;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  const unsigned long long my_recv = stage + c.rank * c.slice_cap;
  for (unsigned long long v0 = first; v0 < V; v0 += stride * U) {
    F8 x[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj) {
        // element v * 8 of block j, addressed from the start of `in` / of this launch's part of the bucket
        const unsigned long long jb = slice_of<W>(c.rank, jj) * block;
        if (v < V) x[u][jj] = load_src<MODE>(src, in, jb + v * 8, jb + n, buf_aligned<MODE>(static_cast<const Elem*>(in) + jb));
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj)
        if (v < V) st_wire<MODE>(c.peer[jj] + my_recv + v * WVB, compress<MODE>(x[u][jj], scale));
    }
  }
}

// Float SUM / AVG: out <- round(sum_r wire(scale * in_r[rank block])), the rank-order fp32 sum of k_twoshot.
template <int MODE, int W>
__global__ void __launch_bounds__(kThreads, 1)
    k_reduce_scatter(CommDev c, const __grid_constant__ Src src, void* out, const void* in, unsigned long long n,
                     unsigned long long block, float scale) {
  using namespace dev;
  constexpr int WVB = Wire<MODE>::kBytes;
  constexpr int U = vecs_per_trip(W);
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  const unsigned long long V = (n + 7) / 8;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;

  // ---- phase A -------------------------------------------------------------------------------
  rs_scatter<MODE, W>(c, src, in, n, block, scale, stage);
  cta_xbar(c, seq0 * 4u + 1u);

  // ---- phase B -------------------------------------------------------------------------------
  const bool aligned = buf_aligned<MODE>(out);
  const uint8_t* mine = c.peer[0] + stage;
  for (unsigned long long v0 = first; v0 < V; v0 += stride * U) {
    Wire<MODE> w[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
      if (v < V) {
#pragma unroll
        for (int r = 0; r < W; ++r) w[u][r] = ld_wire<MODE>(mine + r * c.slice_cap + v * WVB);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
      if (v < V) {
        const F8 s = reduce_rank_order<MODE, W>(w[u]);
        store_out<MODE>(out, v * 8, n, aligned, finalize<MODE>(s));
      }
    }
  }
  op_end(c);
}

// The same reduce-scatter with the optimizer step as its phase B epilogue (b2_reduce_scatter_step, b2_optim.cuh): the
// reduced vec is rounded as `out` would hold it, then steps this rank's parameter and state slices at the same block
// offset.  Phase B runs one vec per trip: the epilogue's three loads and stores per element need the registers.  The bf16
// bucket's instances (b2_reduce_scatter_step_bf16) step fp32 masters with the bf16-rounded gradient and write the bf16
// parameters next to them.
template <int MODE, int W>
__global__ void __launch_bounds__(kThreads, 1)
    k_reduce_scatter_step(CommDev c, const __grid_constant__ Src src, const __grid_constant__ typename OptOf<MODE>::type o, unsigned long long n,
                          unsigned long long block, float scale) {
  using namespace dev;
  constexpr int WVB = Wire<MODE>::kBytes;
  __shared__ OptCta t;
  const uint64_t seq0 = op_begin(c);
  // stage_of(c, seq0), open-coded: the call moves ptxas's register allocation of 8 instances (modes 0, 1 and 3 at W <= 4)
  const unsigned long long stage = (seq0 & 1u) ? c.stage_off[1] : c.stage_off[0];
  const unsigned long long V = (n + 7) / 8;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  opt_cta_init(o, t);  // visible to every thread after cta_xbar's barriers

  rs_scatter<MODE, W>(c, src, nullptr, n, block, scale, stage);
  cta_xbar(c, seq0 * 4u + 1u);

  const uint8_t* mine = c.peer[0] + stage;
  RunHint h;
  for (unsigned long long v = first; v < V; v += stride) {
    Wire<MODE> w[W];
#pragma unroll
    for (int r = 0; r < W; ++r) w[r] = ld_wire<MODE>(mine + r * c.slice_cap + v * WVB);
    const F8 s = reduce_rank_order<MODE, W>(w);
    opt_step_vec(o, t, h, v * 8, n, widen<MODE>(finalize<MODE>(s)));
  }
  op_end(c);
}

// Integer SUM and MIN / MAX on every dtype: out[i] <- OP over r of in_r[rank block][i], combined in rank order, on raw
// 16-byte vecs (W at run time, as k_reduce_exact).
template <int DT, int OP>
__global__ void __launch_bounds__(kThreads, 1) k_reduce_scatter_exact(CommDev c, void* out, const void* in,
                                                                       unsigned long long n, unsigned long long block) {
  using namespace dev;
  constexpr int E = exact::DtypeTraits<DT>::kBytes;
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  const unsigned long long V = (n * E + 15) / 16;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  const unsigned long long my_recv = stage + c.rank * c.slice_cap;
  for (unsigned long long v = first; v < V; v += stride) {
    uint4 q[B2_MAX_WORLD];
#pragma unroll
    for (int jj = 0; jj < B2_MAX_WORLD; ++jj) {
      if (jj < c.world) {
        const uint8_t* src = static_cast<const uint8_t*>(in) + rank_at(c, jj) * block * E;  // the block that goes to peer[jj]
        q[jj] = exact::ld_local<E>(src, (reinterpret_cast<uintptr_t>(src) & 15u) == 0, v, n);
      }
    }
#pragma unroll
    for (int jj = 0; jj < B2_MAX_WORLD; ++jj)
      if (jj < c.world) stg_u4(c.peer[jj] + my_recv + v * 16, q[jj]);
  }
  cta_xbar(c, seq0 * 4u + 1u);
  uint8_t* p = static_cast<uint8_t*>(out);
  const bool aligned = (reinterpret_cast<uintptr_t>(out) & 15u) == 0;
  const uint8_t* mine = c.peer[0] + stage;
  for (unsigned long long v = first; v < V; v += stride) {
    uint4 q[B2_MAX_WORLD];
#pragma unroll
    for (int r = 0; r < B2_MAX_WORLD; ++r)
      if (r < c.world) q[r] = ldg_u4(mine + r * c.slice_cap + v * 16);
    uint4 acc = q[0];
#pragma unroll
    for (int r = 1; r < B2_MAX_WORLD; ++r)
      if (r < c.world) acc = exact::combine<DT, OP>(acc, q[r]);
    exact::st_local<E>(p, aligned, v, n, acc);
  }
  op_end(c);
}
