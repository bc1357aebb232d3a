// b2_reduce.cuh — reduce to a root (b2_reduce): the root's tensor ends with the allreduce of the W ranks' tensors, and
// every other rank's tensor is only read.  A reduce-scatter whose reduced blocks only the root pulls:
//   A  push-scatter : slice j of my message -> recv[me] of rank j (raw vecs, or wire(scale * x) for a float sum)
//   B  reduce       : combine recv[0..W-1] of my own slice in rank order, write my "reduced" region
//   C  pull (root)  : LOAD slice j from rank j's "reduced" region over NVLink, widen, write the root's tensor
// Two cta_xbar between them.  Phases A and B are k_twoshot's (float SUM / AVG) or k_reduce_exact's combine (integer SUM,
// MIN / MAX) on k_twoshot's slices, regions and flag phases, so the root ends with the bits the allreduce leaves there.
// Traffic per rank: (W-1)/W * S out in phase A; the root takes in another (W-1)/W * S in phase C.  A non-root is done
// after the second barrier, before the root has read its "reduced" region: DESIGN.md 2.2 says why it cannot overwrite it
// too early.
#pragma once

#include "b2_dev.cuh"
#include "b2_exact.cuh"

// Float SUM / AVG: buf <- round(sum_r wire(scale * buf_r)) on the root, in rank order.  n elements in W slices of Ls vecs.
template <int MODE, int W>
__global__ void __launch_bounds__(kThreads, 1)
    k_reduce(CommDev c, void* buf, unsigned long long n, float scale, int root) {
  using namespace dev;
  constexpr int WVB = Wire<MODE>::kBytes;
  constexpr int U = vecs_per_trip(W);
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  const bool aligned = buf_aligned<MODE>(buf);
  const unsigned long long V = (n + 7) / 8;
  const unsigned long long Ls = (V + W - 1) / W;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  const unsigned long long my_recv = stage + c.rank * c.slice_cap;
  const unsigned long long reduced = stage + static_cast<unsigned long long>(W) * c.slice_cap;

  // ---- phase A: push-scatter -------------------------------------------------------------------
  for (unsigned long long v0 = first; v0 < Ls; v0 += stride * U) {
    F8 x[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj) {
        const unsigned long long gv = slice_of<W>(c.rank, jj) * Ls + v;
        if (v < Ls && gv < V) x[u][jj] = load_in<MODE>(buf, gv * 8, n, aligned);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj) {
        const unsigned long long gv = slice_of<W>(c.rank, jj) * Ls + v;
        if (v < Ls && gv < V) st_wire<MODE>(c.peer[jj] + my_recv + v * WVB, compress<MODE>(x[u][jj], scale));
      }
    }
  }
  cta_xbar(c, seq0 * 4u + 1u);

  // ---- phase B: reduce my slice into my "reduced" region -----------------------------------------
  uint8_t* mine = c.peer[0];
  const unsigned long long base = c.rank * Ls;
  for (unsigned long long v0 = first; v0 < Ls; v0 += stride * U) {
    Wire<MODE> w[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
      if (v < Ls && base + v < V) {
#pragma unroll
        for (int r = 0; r < W; ++r) w[u][r] = ld_wire<MODE>(mine + stage + r * c.slice_cap + v * WVB);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
      if (v < Ls && base + v < V) {
        const F8 s = reduce_rank_order<MODE, W>(w[u]);
        st_wire<MODE>(mine + reduced + v * WVB, finalize<MODE>(s));
      }
    }
  }
  cta_xbar(c, seq0 * 4u + 2u);

  // ---- phase C: the root pulls every slice ---------------------------------------------------------
  if (c.rank == root) {
    for (unsigned long long v0 = first; v0 < Ls; v0 += stride * U) {
      Wire<MODE> w[U][W];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const unsigned long long v = v0 + u * stride;
#pragma unroll
        for (int jj = 0; jj < W; ++jj) {
          const unsigned long long gv = slice_of<W>(c.rank, jj) * Ls + v;
          if (v < Ls && gv < V) w[u][jj] = ld_wire<MODE>(c.peer[jj] + reduced + v * WVB);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const unsigned long long v = v0 + u * stride;
#pragma unroll
        for (int jj = 0; jj < W; ++jj) {
          const unsigned long long gv = slice_of<W>(c.rank, jj) * Ls + v;
          if (v < Ls && gv < V) store_out<MODE>(buf, gv * 8, n, aligned, w[u][jj]);
        }
      }
    }
  }
  op_end(c);
}

// Integer SUM and MIN / MAX on every dtype: buf <- OP over r of buf_r on the root, combined in rank order, on raw 16-byte
// vecs (W at run time, as k_reduce_exact).  n elements in W slices of Ls vecs.
template <int DT, int OP>
__global__ void __launch_bounds__(kThreads, 1) k_reduce_exact_root(CommDev c, void* buf, unsigned long long n, int root) {
  using namespace dev;
  constexpr int E = exact::DtypeTraits<DT>::kBytes;
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  uint8_t* p = static_cast<uint8_t*>(buf);
  const bool aligned = (reinterpret_cast<uintptr_t>(buf) & 15u) == 0;
  const unsigned long long V = (n * E + 15) / 16;
  const unsigned long long Ls = (V + c.world - 1) / c.world;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  const unsigned long long my_recv = stage + c.rank * c.slice_cap;
  const unsigned long long reduced = stage + static_cast<unsigned long long>(c.world) * c.slice_cap;

  // ---- phase A ----
  for (unsigned long long v = first; v < Ls; v += stride) {
    uint4 q[B2_MAX_WORLD];
#pragma unroll
    for (int jj = 0; jj < B2_MAX_WORLD; ++jj) {
      const unsigned long long gv = rank_at(c, jj) * Ls + v;
      if (jj < c.world && gv < V) q[jj] = exact::ld_local<E>(p, aligned, gv, n);
    }
#pragma unroll
    for (int jj = 0; jj < B2_MAX_WORLD; ++jj) {
      const unsigned long long gv = rank_at(c, jj) * Ls + v;
      if (jj < c.world && gv < V) stg_u4(c.peer[jj] + my_recv + v * 16, q[jj]);
    }
  }
  cta_xbar(c, seq0 * 4u + 1u);

  // ---- phase B ----
  uint8_t* mine = c.peer[0];
  const unsigned long long base = c.rank * Ls;
  for (unsigned long long v = first; v < Ls && base + v < V; v += stride) {
    uint4 q[B2_MAX_WORLD];
#pragma unroll
    for (int r = 0; r < B2_MAX_WORLD; ++r)
      if (r < c.world) q[r] = ldg_u4(mine + stage + r * c.slice_cap + v * 16);
    uint4 acc = q[0];
#pragma unroll
    for (int r = 1; r < B2_MAX_WORLD; ++r)
      if (r < c.world) acc = exact::combine<DT, OP>(acc, q[r]);
    stg_u4(mine + reduced + v * 16, acc);
  }
  cta_xbar(c, seq0 * 4u + 2u);

  // ---- phase C (root) ----
  if (c.rank == root) {
    for (unsigned long long v = first; v < Ls; v += stride) {
      uint4 q[B2_MAX_WORLD];
#pragma unroll
      for (int jj = 0; jj < B2_MAX_WORLD; ++jj) {
        const unsigned long long gv = rank_at(c, jj) * Ls + v;
        if (jj < c.world && gv < V) q[jj] = ldg_u4(c.peer[jj] + reduced + v * 16);
      }
#pragma unroll
      for (int jj = 0; jj < B2_MAX_WORLD; ++jj) {
        const unsigned long long gv = rank_at(c, jj) * Ls + v;
        if (jj < c.world && gv < V) exact::st_local<E>(p, aligned, gv, n, q[jj]);
      }
    }
  }
  op_end(c);
}
