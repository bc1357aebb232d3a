// b2_pipe.cuh — chunk-pipelined, warp-specialised allreduce kernels.
//
// Why: in the single-pass two-shot kernel (b2_kernels.cuh) every CTA runs scatter -> barrier -> reduce -> barrier -> gather
// in lock step, so the NVLink phases, the HBM-only phases and the barriers (release fence = drain of every
// outstanding remote store, flag round trip) add up: at a 25 MiB DDP bucket and W = 8 a large part of the collective is
// not wire time.  Here the message is cut into K chunks and the CTA into three ROLE GROUPS of
// warps that run the three phases of DIFFERENT chunks at the same time and never synchronise with each other inside the
// CTA - the only dependencies are the cross-rank ones, carried by per-(CTA index, kind, chunk) flag words:
//
//   NVLS  (k_pipe<.., kNvls>; needs the multicast mapping of the arena):
//     A cast   : read my fp32 bucket once, cast+scale, store bf16 into MY stage (local HBM/L2)        -> signal X1[k]
//     B move   : wait X1[k] from all ranks; multimem.ld_reduce my slice (the SWITCH sums the W stages, fp32 accumulate,
//                one rounding) and multimem.st the result into every rank's OUTPUT buffer          -> un-fenced hint X2[k]
//     C widen  : wait for the hint; read my output buffer (all W slices), validating every vec against the SENTINEL the
//                buffer is kept filled with (a vec is there when it no longer holds the sentinel: no release fence, no
//                second barrier - the drain of the multicast stores disappears from the critical path), widen,
//                write my bucket, put the sentinel back
//     NVLink traffic per GPU and direction: (1 + 1/W) * S instead of the 2 (W-1)/W * S of any P2P algorithm.
//
//   P2P   (k_pipe<.., kP2p>; any world, plain peer mappings):
//     A scatter: read my bucket once, cast+scale, STORE slice j into rank j's recv[me]                -> signal X1[k]
//     B reduce : wait X1[k]; sum recv[0..W-1] of my slice in rank order (fp32), round once -> "reduced" -> signal X2[k]
//     C gather : wait X2[k]; LOAD slice j from rank j's "reduced", widen, write my bucket
//
// Signalling is DECOUPLED from data movement.  A release (MEMBAR.SYS: drain of the outstanding stores, microseconds after a
// burst of NVLink stores) executed by a data warp stalls that warp and, at the next group barrier, its whole role - once
// per chunk, enough to make the pipelined kernel slower than the single-pass one.  So roles A
// and B each own one SIGNALLER warp that moves no data: the data warps finish chunk k with a barrier among themselves and a
// shared-memory mailbox store (st.release.cta), and carry on with chunk k+1; the signaller polls the mailbox
// (ld.acquire.cta) and publishes chunk k to every rank with st.release.sys.  Waiting stays with the data warps
// (ld.acquire.sys by their first W threads, then the group barrier): an acquire drains nothing.  Chunk (k, b) = vecs [(k*g + b) * cell, +cell) of every slice
// (g = grid size): chunk-major, so the bytes of one pipeline step are contiguous bands of each slice, and CTA b of every
// rank touches exactly the same vec indices - the only cross-rank dependencies are between equal CTA indices, so neither
// a grid-wide sync nor co-residency of a rank's own CTAs is needed.
//
// Staging-buffer reuse across collectives is safe for the same reason as in the single-pass kernels (DESIGN.md 2.1):
// the two stages alternate by the parity of the device-resident op counter, and collective n+2 can only start once every
// CTA of collective n+1 has passed its X2 waits, which peers signal only after their collective n has completed.
#pragma once

#include "b2_dev.cuh"

namespace pl {

enum { kNvls = 0, kP2p = 1 };

// Warp roles (threads): A = cast/scatter (kAD data threads + one signaller warp), B = move/reduce (kBD + one signaller
// warp), C = widen/gather.
constexpr int kAD = 160, kBD = 96, kCD = 192, kSig = 32;
constexpr int kA0 = 0, kAS = kA0 + kAD, kB0 = kAS + kSig, kBS = kB0 + kBD, kC0 = kBS + kSig;
static_assert(kC0 + kCD == kThreads, "roles must tile the CTA");
static_assert(kAD % 32 == 0 && kBD % 32 == 0 && kCD % 32 == 0, "roles are whole warps");

__device__ __forceinline__ void group_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void mail_post(uint32_t* box, uint32_t v) {
  asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(box))), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t mail_peek(const uint32_t* box) {
  uint32_t v;
  asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(static_cast<uint32_t>(__cvta_generic_to_shared(box))) : "memory");
  return v;
}

__device__ __forceinline__ uint64_t* flag_slot(uint8_t* arena, const CommDev& c, int kind, int k) {
  const size_t idx = (static_cast<size_t>(blockIdx.x) * kPipeKinds + kind) * kMaxChunks + k;
  return reinterpret_cast<uint64_t*>(arena + c.pflag_off + idx * kFlagSlotBytes);
}

// Data side: the `count` data threads of a role have issued their stores for chunk k.
__device__ __forceinline__ void chunk_done(int id, int count, int t, uint32_t* box, int k) {
  group_sync(id, count);                                  // every data thread's stores are ordered before the post below
  if (t == 0) mail_post(box, static_cast<uint32_t>(k + 1));
}
// Signaller warp of a role: publish chunks 0..nk-1 of `kind` to every rank as the data warps complete them.
// Lane l (< world) pairs with rank (rank + l) % world and writes word [my rank] of that rank's slot.  ONE release fence
// covers every chunk the data warps have finished by the time the signaller looks (a fence after a burst of stores waits
// for the drain of the memory system's backlog, and fences of one warp do not overlap): the pipeline granularity
// adapts to the fence latency instead of serialising K fences.
template <bool FENCE>
__device__ __forceinline__ void signaller(const CommDev& c, int lane, const uint32_t* box, int kind, int nk, uint64_t seq) {
  int k = 0;
  while (k < nk) {
    unsigned long long t0 = 0;
    unsigned spins = 0;
    uint32_t done;
    while ((done = mail_peek(box)) < static_cast<uint32_t>(k + 1)) {  // chunk k not finished by the data warps yet
      if ((++spins & 1023u) == 0) {
        const unsigned long long now = dev::globaltimer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > c.timeout_ns) {  // the data warps are stuck behind a dead peer: they report it themselves
          done = static_cast<uint32_t>(nk);
          break;
        }
      }
    }
    __syncwarp();
    if (lane < c.world) {
      // everything the data warps stored for chunks < done is ordered first - unless the flag is only a HINT (NVLS X2: the
      // consumer validates every vec against the sentinel itself, the flag just tells it when polling becomes worthwhile)
      if constexpr (FENCE) asm volatile("fence.acq_rel.sys;" ::: "memory");
      uint8_t* their = dev::peer_sel(c, lane);
      for (int kk = k; kk < static_cast<int>(done); ++kk)
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(flag_slot(their, c, kind, kk) + c.rank), "l"(seq) : "memory");
    }
    k = static_cast<int>(done);
  }
}
// Wait until every rank has published `seq` for (kind, k): thread t (< world) polls word [t] of my own slot.
__device__ __forceinline__ void group_wait(const CommDev& c, int id, int count, int t, int kind, int k, uint64_t seq) {
  if (t < c.world) dev::wait_flag(c, flag_slot(c.peer[0], c, kind, k) + t, seq);
  group_sync(id, count);  // peers' data is now visible to every thread of the group (the acquire invalidated L1)
}

}  // namespace pl

template <int MODE, int W, int ALG>
__global__ void __launch_bounds__(kThreads, 1)
    k_pipe(CommDev c, const __grid_constant__ Src src, void* buf, unsigned long long n, float scale, int K, unsigned long long cell) {
  using namespace dev;
  using namespace pl;
  constexpr int WVB = Wire<MODE>::kBytes;
  constexpr int U = vecs_per_trip(W);
  __shared__ uint32_t mail[2];  // [0]: chunks role A has finished, [1]: chunks role B has finished
  const uint64_t seq0 = op_begin(c);
  const uint64_t seq = seq0 * 4u + 1u;
  const unsigned long long stage = stage_of(c, seq0);
  const bool aligned = buf_aligned<MODE>(buf);
  const unsigned long long V = (n + 7) / 8;
  const unsigned long long Ls = (V + W - 1) / W;
  const unsigned long long g = gridDim.x, b = blockIdx.x;
  const unsigned long long reduced = stage + static_cast<unsigned long long>(W) * c.slice_cap;  // P2P only
  const unsigned long long nvls_out = ((seq0 & 1u) ? c.ll_off[1] : c.ll_off[0]) + static_cast<unsigned long long>(W) * c.slice_cap;  // NVLS only: "out" regions
  uint8_t* const mine = c.peer[0];
  const int tid = threadIdx.x;
  // chunks this CTA really has: cell (k, b) starts at (k*g + b)*cell, empty from the first k with start >= Ls on
  int nk = 0;
  while (nk < K && (static_cast<unsigned long long>(nk) * g + b) * cell < Ls) ++nk;
  if (tid < 2) mail[tid] = 0;
  __syncthreads();

  if (tid < kAS) {
    // ================= role A data: cast (NVLS) / scatter (P2P) =================
    const int t = tid - kA0;
      if (t == 0) trace_stamp(c, 0);
    for (int k = 0; k < nk; ++k) {
      const unsigned long long lo = (static_cast<unsigned long long>(k) * g + b) * cell;
      const unsigned long long hi = lo + cell < Ls ? lo + cell : Ls;
      for (unsigned long long v0 = lo + t; v0 < hi; v0 += static_cast<unsigned long long>(kAD) * U) {
        F8 x[U][W];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kAD;
#pragma unroll
          for (int jj = 0; jj < W; ++jj) {
            const int j = slice_of<W>(c.rank, jj);
            const unsigned long long gv = j * Ls + v;
            if (v < hi && gv < V) x[u][jj] = load_src<MODE>(src, buf, gv * 8, n, aligned);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kAD;
#pragma unroll
          for (int jj = 0; jj < W; ++jj) {
            const int j = slice_of<W>(c.rank, jj);
            const unsigned long long gv = j * Ls + v;
            if (v < hi && gv < V) {
              const Wire<MODE> w = compress<MODE>(x[u][jj], scale);
              if constexpr (ALG == kNvls)
                st_wire<MODE>(mine + stage + gv * WVB, w);  // my stage: one message-sized buffer, vec gv at gv
              else
                st_wire<MODE>(c.peer[jj] + stage + c.rank * c.slice_cap + v * WVB, w);  // rank j's recv[me]
            }
          }
        }
      }
      chunk_done(1, kAD, t, &mail[0], k);
    }
    if (t == 0) trace_stamp(c, 1);
  } else if (tid < kB0) {
    signaller<true>(c, tid - kAS, &mail[0], 0, nk, seq);  // role A's signaller: X1[k]
  } else if (tid < kBS) {
    // ================= role B data: move (NVLS) / reduce (P2P) =================
    const int t = tid - kB0;
    const unsigned long long base = c.rank * Ls;  // my slice
    for (int k = 0; k < nk; ++k) {
      const unsigned long long lo = (static_cast<unsigned long long>(k) * g + b) * cell;
      const unsigned long long hi = lo + cell < Ls ? lo + cell : Ls;
      group_wait(c, 2, kBD, t, 0, k, seq);
      if (t == 0 && k == 0) trace_stamp(c, 2);
      if constexpr (ALG == kNvls) {
        constexpr int UM = kF32Wire<MODE> ? 4 : 8;  // 128 B of switch-side reductions in flight per thread
        const uint8_t* const mc_in = c.mc + stage;   // every rank's staged contribution, summed by the switch on load
        uint8_t* const mc_out = c.mc + nvls_out + c.rank * c.slice_cap;  // out[me] on every rank, written by the switch on store
        for (unsigned long long v0 = lo + t; v0 < hi; v0 += static_cast<unsigned long long>(kBD) * UM) {
          Wire<MODE> q[UM];
#pragma unroll
          for (int u = 0; u < UM; ++u) {
            const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kBD;
            if (v < hi && base + v < V) q[u] = mm_ld_reduce_wire<MODE>(mc_in + (base + v) * WVB);
          }
#pragma unroll
          for (int u = 0; u < UM; ++u) {
            const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kBD;
            if (v < hi && base + v < V) mm_st_wire<MODE>(mc_out + v * WVB, wire_no_sentinel<MODE>(q[u]));
          }
        }
      } else {
        for (unsigned long long v0 = lo + t; v0 < hi; v0 += static_cast<unsigned long long>(kBD) * U) {
          Wire<MODE> w[U][W];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kBD;
            if (v < hi && base + v < V) {
#pragma unroll
              for (int r = 0; r < W; ++r) w[u][r] = ld_wire<MODE>(mine + stage + r * c.slice_cap + v * WVB);
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kBD;
            if (v < hi && base + v < V) {
              const F8 s = reduce_rank_order<MODE, W>(w[u]);
              st_wire<MODE>(mine + reduced + v * WVB, finalize<MODE>(s));
            }
          }
        }
      }
      chunk_done(2, kBD, t, &mail[1], k);
    }
    if (t == 0) trace_stamp(c, 3);
  } else if (tid < kC0) {
    signaller<ALG != kNvls>(c, tid - kBS, &mail[1], 1, nk, seq);  // role B's signaller: X2[k] (NVLS: un-fenced hint)
  } else {
    // ================= role C: widen (NVLS) / gather (P2P) =================
    const int t = tid - kC0;
    for (int k = 0; k < nk; ++k) {
      const unsigned long long lo = (static_cast<unsigned long long>(k) * g + b) * cell;
      const unsigned long long hi = lo + cell < Ls ? lo + cell : Ls;
      group_wait(c, 3, kCD, t, 1, k, seq);
      if (t == 0 && k == 0) trace_stamp(c, 4);
      for (unsigned long long v0 = lo + t; v0 < hi; v0 += static_cast<unsigned long long>(kCD) * U) {
        Wire<MODE> w[U][W];
        bool pend[U][W];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kCD;
#pragma unroll
          for (int jj = 0; jj < W; ++jj) {
            const int j = slice_of<W>(c.rank, jj);
            const unsigned long long gv = j * Ls + v;
            pend[u][jj] = false;
            if (v < hi && gv < V) {
              if constexpr (ALG == kNvls)
                w[u][jj] = wire_poll<MODE>(mine + nvls_out + j * c.slice_cap + v * WVB, &pend[u][jj]);  // out[j]: multicast by the switch
              else
                w[u][jj] = ld_wire<MODE>(c.peer[jj] + reduced + v * WVB);  // rank j's reduced slice, over NVLink
            }
          }
        }
        if constexpr (ALG == kNvls) {
          // data the hint ran ahead of: poll until the sentinel is gone (bounded like every other wait)
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kCD;
#pragma unroll
            for (int jj = 0; jj < W; ++jj) {
              if (!pend[u][jj]) continue;
              const int j = slice_of<W>(c.rank, jj);
              wait_wire<MODE, 64, 64>(c, mine + nvls_out + j * c.slice_cap + v * WVB, w[u][jj]);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kCD;
#pragma unroll
          for (int jj = 0; jj < W; ++jj) {
            const int j = slice_of<W>(c.rank, jj);
            const unsigned long long gv = j * Ls + v;
            if (v < hi && gv < V) {
              store_out<MODE>(buf, gv * 8, n, aligned, w[u][jj]);
              if constexpr (ALG == kNvls) wire_reset<MODE>(mine + nvls_out + j * c.slice_cap + v * WVB);  // back to "not written yet"
            }
          }
        }
      }
    }
    if (t == 0) trace_stamp(c, 5);
  }
  op_end(c);
}
