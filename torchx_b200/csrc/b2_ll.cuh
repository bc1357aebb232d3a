// b2_ll.cuh — barrier-free two-shot allreduce ("LL two-shot"): every synchronisation is carried by the data itself.
//
// Why: the single-pass two-shot kernel spends a sizeable share of a DDP-bucket collective in its two flag barriers - each
// one a release fence that has to drain the memory system's backlog of NVLink stores plus a flag round trip - and the
// pull-gather cannot start before the slowest rank has
// passed the second one.  Chunk pipelining hides little of it (the fences of one warp serialise; b2_pipe.cuh).  Here there
// is no flag and no fence on the data path at all:
//
//   1  push-scatter : read my bucket once, cast+scale, STORE slice j into rank j's recv[me]              (NVLink egress)
//   2  reduce+push  : poll MY recv[0..W-1] for my slice until every 32-bit word has arrived, fp32 accumulate in rank
//                     order, round once, STORE the reduced slice into out[me] of EVERY rank               (NVLink egress)
//   3  widen        : poll MY out[0..W-1], widen, write my bucket          (local only; interleaved with phase 2, one trip behind)
//
// "Arrived" = the word no longer holds the SENTINEL the buffers are kept filled with (kSentinel: a NaN pattern that the
// producers canonicalise away, so data never contains it).  Each 4-byte word is validated on its own, so no assumption
// about the atomicity of wider NVLink stores is needed.  A consumer puts the sentinel back right after reading; the two
// parities of the op counter double-buffer the regions, and a one-word-per-peer flow-control flag (published at kernel
// START, where the stream order already guarantees the previous collective's stores are done - no fence) keeps a fast
// rank from writing a region before its owner has left the collective that last used it.
// Every transfer is a push (fire-and-forget stores; nothing ever waits for a remote load), every wait is a poll of local
// L2, and the three phases of different vec indices overlap freely across threads: thread t of rank i only ever depends on
// thread t of the other ranks.  The arithmetic is exactly the single-pass kernel's (rank-order fp32 accumulate, one
// rounding): results are bit-identical to the oracle.
#pragma once

#include "b2_dev.cuh"

template <int MODE, int W>
__global__ void __launch_bounds__(kThreads, 1)
    k_ll(CommDev c, const __grid_constant__ Src src, void* buf, unsigned long long n, float scale) {
  using namespace dev;
  constexpr int WVB = Wire<MODE>::kBytes;
  constexpr int U = vecs_per_trip(W);
  const uint64_t seq0 = op_begin(c);
  const unsigned long long base_ll = (seq0 & 1u) ? c.ll_off[1] : c.ll_off[0];
  const bool aligned = buf_aligned<MODE>(buf);
  const unsigned long long V = (n + 7) / 8;
  const unsigned long long Ls = (V + W - 1) / W;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  uint8_t* const mine = c.peer[0];
  const unsigned long long my_recv = base_ll + c.rank * c.slice_cap;                                        // recv[me] on a peer
  const unsigned long long my_out = base_ll + (static_cast<unsigned long long>(W) + c.rank) * c.slice_cap;  // out[me] on a peer
  if (threadIdx.x == 0) trace_stamp(c, 0);

  // ---- flow control: tell the peers this collective has started here (so everything before it is complete), and do not
  // write a parity's buffers before every peer has at least started the PREVIOUS collective (= left the one before it,
  // the last that can have used this parity)
  if (threadIdx.x < W) {
    const int jj = threadIdx.x;
    const int p = slice_of<W>(c.rank, jj);
    if (blockIdx.x == 0)
      asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(reinterpret_cast<uint64_t*>(peer_sel(c, jj) + c.llflag_off) + c.rank), "l"(seq0)
                   : "memory");
    // the first op has no predecessor: wait for 0, not for seq0 - 1 = 2^64 - 1
    if (jj != 0) wait_flag(c, reinterpret_cast<const uint64_t*>(mine + c.llflag_off) + p, seq0 == 0 ? 0 : seq0 - 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) trace_stamp(c, 1);

  // ---- phase 1: push-scatter ------------------------------------------------------------------
  for (unsigned long long v0 = first; v0 < Ls; v0 += stride * U) {
    F8 x[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj) {
        const int j = slice_of<W>(c.rank, jj);
        const unsigned long long gv = j * Ls + v;
        if (v < Ls && gv < V) x[u][jj] = load_src<MODE>(src, buf, gv * 8, n, aligned);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj) {
        const int j = slice_of<W>(c.rank, jj);
        const unsigned long long gv = j * Ls + v;
        if (v < Ls && gv < V)
          st_wire<MODE>(c.peer[jj] + my_recv + v * WVB, wire_no_sentinel<MODE>(compress<MODE>(x[u][jj], scale)));
      }
    }
  }
  if (threadIdx.x == 0) trace_stamp(c, 2);

  // ---- phases 2 and 3, interleaved: in trip i a thread reduces + pushes its vecs of trip i (NVLink egress) and widens
  // the vecs of trip i-1 (local L2/HBM only), whose slices the peers pushed one trip ago - so the final local pass hides
  // behind the pushes instead of following them (for a 256 MiB bucket that is half a gigabyte of HBM traffic).  No cycle: widening
  // trip k needs the peers' pushes of trip k, which they issue before they widen trip k-1.
  {
    const unsigned long long base = c.rank * Ls;
    const unsigned long long step = stride * U;
    for (unsigned long long v0 = first;; v0 += step) {
      const bool do2 = v0 < Ls;
      const bool do3 = v0 >= step + first && v0 - step < Ls;
      if (!do2 && !do3) break;
      if (do2) {  // ---- phase 2: reduce my slice as its contributions arrive, push the result to everyone
        // G contributions of one vec are polled together (all W for the 16-byte bf16 / fp16 wire vecs; 4 for the 32-byte fp32
        // ones, which would not fit the register file otherwise); accumulation stays in rank order either way.
        constexpr int G = (kF32Wire<MODE> && W > 4) ? 4 : W;
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const unsigned long long v = v0 + u * stride;
          if (v < Ls && base + v < V) {
            F8 s;
#pragma unroll
            for (int r0 = 0; r0 < W; r0 += G) {
              Wire<MODE> w[G];
              bool pend[G];
#pragma unroll
              for (int g = 0; g < G; ++g)
                if (r0 + g < W) w[g] = wire_poll<MODE>(mine + base_ll + (r0 + g) * c.slice_cap + v * WVB, &pend[g]);
#pragma unroll
              for (int g = 0; g < G; ++g) {
                if (r0 + g < W) {
                  uint8_t* p = mine + base_ll + (r0 + g) * c.slice_cap + v * WVB;
                  if (pend[g]) wait_wire<MODE, 40, 128>(c, p, w[g]);
                  wire_reset<MODE>(p);  // back to "not written yet" for the collective after next
                  if (r0 + g == 0) s = widen<MODE>(w[g]);
                  else accumulate(s, widen<MODE>(w[g]));  // rank order, fp32
                }
              }
            }
            const Wire<MODE> q = wire_no_sentinel<MODE>(finalize<MODE>(s));
#pragma unroll
            for (int jj = 0; jj < W; ++jj) st_wire<MODE>(c.peer[jj] + my_out + v * WVB, q);
          }
        }
      }
      if (do3) {  // ---- phase 3: widen every slice of the previous trip as it arrives
        const unsigned long long p0 = v0 - step;
        constexpr int G = (kF32Wire<MODE> && W > 4) ? 4 : W;
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const unsigned long long v = p0 + u * stride;
#pragma unroll
          for (int j0 = 0; j0 < W; j0 += G) {
            Wire<MODE> w[G];
            bool pend[G];
#pragma unroll
            for (int g = 0; g < G; ++g) {
              // slice_of<W>(c.rank, j0 + g), open-coded: the call moves ptxas's register allocation of k_ll at W = 3, 5,
              // 6, 7 and 8 (spills appear or disappear), so both phase-3 rotations keep this form
              int j = c.rank + j0 + g;
              if (j >= W) j -= W;
              pend[g] = false;
              if (j0 + g < W && v < Ls && j * Ls + v < V)
                w[g] = wire_poll<MODE>(mine + base_ll + (static_cast<unsigned long long>(W) + j) * c.slice_cap + v * WVB, &pend[g]);
            }
#pragma unroll
            for (int g = 0; g < G; ++g) {
              int j = c.rank + j0 + g;
              if (j >= W) j -= W;
              const unsigned long long gv = j * Ls + v;
              if (j0 + g < W && v < Ls && gv < V) {
                uint8_t* p = mine + base_ll + (static_cast<unsigned long long>(W) + j) * c.slice_cap + v * WVB;
                if (pend[g]) wait_wire<MODE, 40, 128>(c, p, w[g]);
                store_out<MODE>(buf, gv * 8, n, aligned, w[g]);
                wire_reset<MODE>(p);
              }
            }
          }
        }
      }
    }
  }
  if (threadIdx.x == 0) trace_stamp(c, 5);
  op_end(c);
}
