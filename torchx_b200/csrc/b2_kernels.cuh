// b2_kernels.cuh — the single-pass kernels: W==1 local pass (plain and TMA-staged), one-shot and two-shot allreduce,
// broadcast, barrier.  The chunk-pipelined kernels (NVLS and P2P) live in b2_pipe.cuh.
#pragma once

#include "b2_dev.cuh"
#include "b2_optim.cuh"

// W == 1 (and the single-GPU roofline probe): x <- round(wire(scale * x)), one streaming pass.  Each CTA owns a contiguous
// range of vecs and a thread's successive vecs are 512 apart (a warp still reads 1 KiB of consecutive memory per access):
// when the input comes through a segment table (zero-copy bucket fill) a thread then stays inside one parameter for many
// trips and its segment hint keeps hitting.
template <int MODE>
__global__ void __launch_bounds__(kThreads) k_local_pass(const __grid_constant__ Src src, void* buf, unsigned long long n, float scale) {
  using namespace dev;
  const bool aligned = buf_aligned<MODE>(buf);
  const unsigned long long V = (n + 7) / 8;
  constexpr int U = 4;
  constexpr unsigned long long kTrip = static_cast<unsigned long long>(kThreads) * U;
  const unsigned long long per_cta = (V + gridDim.x - 1) / gridDim.x;
  const unsigned long long span = (per_cta + kTrip - 1) / kTrip * kTrip;
  const unsigned long long lo = blockIdx.x * span;
  const unsigned long long hi = lo + span < V ? lo + span : V;
  SegHint hint;
  for (unsigned long long v0 = lo + threadIdx.x; v0 < hi; v0 += kTrip) {
    F8 x[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kThreads;
      if (v < hi) x[u] = load_src<MODE>(src, hint, buf, v * 8, n, aligned);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + static_cast<unsigned long long>(u) * kThreads;
      if (v < hi) {
        const Wire<MODE> c = compress<MODE>(x[u], scale);
        store_out<MODE>(buf, v * 8, n, aligned, finalize<MODE>(widen<MODE>(c)));
      }
    }
  }
}

// W == 1 with the optimizer step (b2_reduce_scatter_step): the local pass's rounding of each vec read through the segment
// table (mode 0 is not a copy: it rounds to bf16), then the optimizer epilogue on the parameter and state slices
// (b2_optim.cuh) instead of the store.  The local pass's CTA layout, so a thread's segment and run hints keep hitting.
template <int MODE>
__global__ void __launch_bounds__(kThreads, 1) k_local_step(const __grid_constant__ Src src, const __grid_constant__ OptDev o,
                                                         unsigned long long n, float scale) {
  using namespace dev;
  __shared__ OptCta t;
  opt_cta_init(o, t);
  __syncthreads();
  const unsigned long long V = (n + 7) / 8;
  constexpr unsigned long long kTrip = static_cast<unsigned long long>(kThreads) * 4;
  const unsigned long long per_cta = (V + gridDim.x - 1) / gridDim.x;
  const unsigned long long span = (per_cta + kTrip - 1) / kTrip * kTrip;
  const unsigned long long lo = blockIdx.x * span;
  const unsigned long long hi = lo + span < V ? lo + span : V;
  SegHint hint;
  RunHint rh;
  for (unsigned long long v = lo + threadIdx.x; v < hi; v += kThreads) {
    const F8 x = load_src<MODE>(src, hint, nullptr, v * 8, n, false);
    const Wire<MODE> c = compress<MODE>(x, scale);
    opt_step_vec(o, t, rh, v * 8, n, widen<MODE>(finalize<MODE>(widen<MODE>(c))));
  }
}

// ---- TMA building blocks (cp.async.bulk + mbarrier; SASS UBLKCP) ------------------------------------------------
// One elected thread issues bulk copies global -> shared that complete on an mbarrier: the bytes in flight cost no
// registers and no warps, which is what lets a few warps keep a whole SM's share of HBM bandwidth busy.
namespace tma {

constexpr int kTileBytes = 16 << 10;
constexpr int kStages = 4;
constexpr int kTmaThreads = 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// x <- round(wire(scale * x)) on one 16-byte group (4 fp32 or 8 16-bit elements), same arithmetic as compress+finalize.
template <int MODE>
__device__ __forceinline__ uint4 round16(uint4 q, float scale) {
  using namespace dev;
  if constexpr (k16BitBucket<MODE>) {
    uint32_t in[4] = {q.x, q.y, q.z, q.w}, out[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = pack16<MODE>(__fmul_rn(lo16<MODE>(in[i]), scale), __fmul_rn(hi16<MODE>(in[i]), scale));
    return make_uint4(out[0], out[1], out[2], out[3]);
  } else {
    float f[4] = {__uint_as_float(q.x), __uint_as_float(q.y), __uint_as_float(q.z), __uint_as_float(q.w)};
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      if constexpr (kF32Wire<MODE>) {
        o[i] = __float_as_uint(__fmul_rn(f[i], scale));
        o[i + 1] = __float_as_uint(__fmul_rn(f[i + 1], scale));
      } else {
        static_assert(ModeTraits<MODE>::kCastIn, "an fp32 bucket on a 16-bit wire is rounded to the wire format first");
        const uint32_t p = pack16<MODE>(f[i], f[i + 1]);                                            // .to(bf16 / fp16)
        const uint32_t r = pack16<MODE>(__fmul_rn(lo16<MODE>(p), scale), __fmul_rn(hi16<MODE>(p), scale));  // .div_(W)
        if constexpr (ModeTraits<MODE>::kWire == WireFmt::kBF16) {
          o[i] = r << 16;             // widen back to fp32: bf16 bits in the high half
          o[i + 1] = r & 0xffff0000u;
        } else {
          o[i] = __float_as_uint(lo16<MODE>(r));  // widen back to fp32 (exact)
          o[i + 1] = __float_as_uint(hi16<MODE>(r));
        }
      }
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace tma

// TMA-staged variant of the local pass: persistent CTAs stream 16 KiB tiles through a 4-deep shared-memory ring; all
// threads round the tile in place in shared memory, and the tile goes back with a bulk store (shared -> global).
template <int MODE>
__global__ void __launch_bounds__(tma::kTmaThreads) k_local_pass_tma(void* buf, unsigned long long n, float scale) {
  using namespace tma;
  extern __shared__ __align__(128) uint8_t ring_raw[];  // kStages * kTileBytes of dynamic shared memory
  uint8_t(*ring)[kTileBytes] = reinterpret_cast<uint8_t(*)[kTileBytes]>(ring_raw);
  __shared__ alignas(8) uint64_t full[kStages];
  constexpr int kElem = ModeTraits<MODE>::kElemBytes;
  const unsigned long long bytes = n * kElem;
  const unsigned long long ntiles = bytes / kTileBytes;  // full tiles go through TMA; the tail is handled below
  uint8_t* base = static_cast<uint8_t*>(buf);
  const unsigned long long my_first = blockIdx.x;
  const unsigned long long step = gridDim.x;
  const unsigned long long my_count = my_first < ntiles ? (ntiles - my_first + step - 1) / step : 0;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      if (static_cast<unsigned long long>(s) < my_count) {
        mbar_arrive_expect_tx(&full[s], kTileBytes);
        bulk_g2s(ring[s], base + (my_first + s * step) * kTileBytes, kTileBytes, &full[s]);
      }
    }
  }
  for (unsigned long long k = 0; k < my_count; ++k) {
    const int s = static_cast<int>(k % kStages);
    mbar_wait(&full[s], static_cast<uint32_t>((k / kStages) & 1));
    uint4* tile = reinterpret_cast<uint4*>(ring[s]);
#pragma unroll
    for (int i = 0; i < kTileBytes / 16 / kTmaThreads; ++i) {
      const int idx = i * kTmaThreads + threadIdx.x;  // conflict-free: consecutive lanes, consecutive 16 B
      tile[idx] = round16<MODE>(tile[idx], scale);
    }
    fence_proxy_async();  // my generic-proxy writes to the tile are visible to the bulk store (async proxy)
    __syncthreads();
    if (threadIdx.x == 0) {
      bulk_s2g(base + (my_first + k * step) * kTileBytes, ring[s], kTileBytes);
      bulk_commit();
      // Refill the stage whose store was issued ONE iteration ago: allowing one group in flight means that older
      // store has finished reading shared memory, while the store just issued keeps draining.
      if (k >= 1 && k - 1 + kStages < my_count) {
        bulk_wait_read<1>();
        const int sp = static_cast<int>((k - 1) % kStages);
        mbar_arrive_expect_tx(&full[sp], kTileBytes);
        bulk_g2s(ring[sp], base + (my_first + (k - 1 + kStages) * step) * kTileBytes, kTileBytes, &full[sp]);
      }
    }
  }
  if (threadIdx.x == 0) bulk_wait_read<0>();  // shared memory must outlive the last store's reads
  // tail (< 16 KiB): plain loads/stores, spread over the grid
  const unsigned long long tail0 = ntiles * kTileBytes / kElem;
  for (unsigned long long e = tail0 + (static_cast<unsigned long long>(blockIdx.x) * kTmaThreads + threadIdx.x) * 8; e < n;
       e += static_cast<unsigned long long>(gridDim.x) * kTmaThreads * 8) {
    const dev::F8 x = dev::load_in<MODE>(buf, e, n, false);
    const dev::Wire<MODE> c = dev::compress<MODE>(x, scale);
    dev::store_out<MODE>(buf, e, n, false, dev::finalize<MODE>(dev::widen<MODE>(c)));
  }
}

// One-shot: latency regime.  Wire traffic per rank: (W-1) * S out, (W-1) * S in.
template <int MODE, int W>
__global__ void __launch_bounds__(kThreads, 1)
    k_oneshot(CommDev c, const __grid_constant__ Src src, void* buf, unsigned long long n, float scale) {
  using namespace dev;
  constexpr int WVB = Wire<MODE>::kBytes;
  constexpr int U = vecs_per_trip(W);
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  const bool aligned = buf_aligned<MODE>(buf);
  const unsigned long long V = (n + 7) / 8;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (threadIdx.x == 0) trace_stamp(c, 0);

  // phase A: compress my message once, push it into recv[rank] of every rank (mine included)
  for (unsigned long long v0 = first; v0 < V; v0 += stride * U) {
    F8 x[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
      if (v < V) x[u] = load_src<MODE>(src, buf, v * 8, n, aligned);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
      if (v < V) {
        const Wire<MODE> w = compress<MODE>(x[u], scale);
#pragma unroll
        for (int jj = 0; jj < W; ++jj)  // peer[] is rotated: the W ranks never hammer one peer at a time
          st_wire<MODE>(c.peer[jj] + stage + c.rank * c.slice_cap + v * WVB, w);
      }
    }
  }
  if (threadIdx.x == 0) trace_stamp(c, 1);
  cta_xbar(c, seq0 * 4u + 1u);
  if (threadIdx.x == 0) trace_stamp(c, 2);

  // phase B: reduce the W messages (all local now) in rank order, write the caller's tensor
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
        store_out<MODE>(buf, v * 8, n, aligned, finalize<MODE>(reduce_rank_order<MODE, W>(w[u])));
      }
    }
  }
  if (threadIdx.x == 0) trace_stamp(c, 3);
  op_end(c);
}

// Two-shot, single pass: bandwidth regime for worlds / sizes the pipelined kernels do not take.  The message is cut into
// W slices of Ls vecs; rank i owns slice i.
//   A  push-scatter : read my fp32 bucket once, cast+scale, STORE slice j into rank j's recv[me]
//   B  reduce       : sum recv[0..W-1] of my slice (local HBM), fp32 accumulate in rank order,
//                     round once, write my "reduced" region
//   C  pull-gather  : LOAD slice j from rank j's "reduced" region over NVLink, widen, write bucket
// Wire traffic per rank and direction: 2 * (W-1)/W * S  (the allreduce lower bound for P2P).
// CTA b touches the same vec indices of a slice on every rank and in every phase, so the only
// synchronisation needed is among the CTAs with equal blockIdx.x across ranks (no grid sync).
template <int MODE, int W>
__global__ void __launch_bounds__(kThreads, 1)
    k_twoshot(CommDev c, const __grid_constant__ Src src, void* buf, unsigned long long n, float scale) {
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
  if (threadIdx.x == 0) trace_stamp(c, 0);

  // ---- phase A -------------------------------------------------------------------------------
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
          st_wire<MODE>(c.peer[jj] + my_recv + v * WVB, compress<MODE>(x[u][jj], scale));
      }
    }
  }
  if (threadIdx.x == 0) trace_stamp(c, 1);
  cta_xbar(c, seq0 * 4u + 1u);
  if (threadIdx.x == 0) trace_stamp(c, 2);

  // ---- phase B -------------------------------------------------------------------------------
  {
    uint8_t* mine = c.peer[0];
    const unsigned long long base = c.rank * Ls;
    for (unsigned long long v0 = first; v0 < Ls; v0 += stride * U) {
      Wire<MODE> w[U][W];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const unsigned long long v = v0 + u * stride;
        if (v < Ls && base + v < V) {
#pragma unroll
          for (int r = 0; r < W; ++r)
            w[u][r] = ld_wire<MODE>(mine + stage + r * c.slice_cap + v * WVB);
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
  }
  if (threadIdx.x == 0) trace_stamp(c, 3);
  cta_xbar(c, seq0 * 4u + 2u);
  if (threadIdx.x == 0) trace_stamp(c, 4);

  // ---- phase C -------------------------------------------------------------------------------
  for (unsigned long long v0 = first; v0 < Ls; v0 += stride * U) {
    Wire<MODE> w[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj) {
        const int j = slice_of<W>(c.rank, jj);
        const unsigned long long gv = j * Ls + v;
        if (v < Ls && gv < V) w[u][jj] = ld_wire<MODE>(c.peer[jj] + reduced + v * WVB);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long v = v0 + u * stride;
#pragma unroll
      for (int jj = 0; jj < W; ++jj) {
        const int j = slice_of<W>(c.rank, jj);
        const unsigned long long gv = j * Ls + v;
        if (v < Ls && gv < V) store_out<MODE>(buf, gv * 8, n, aligned, w[u][jj]);
      }
    }
  }
  if (threadIdx.x == 0) trace_stamp(c, 5);
  op_end(c);
}

// Broadcast of raw bytes: root pushes into every peer's stage, one barrier, peers copy out.  The stage is always
// addressed in 16-byte vecs (it is aligned on every rank), so CTA b of the root and CTA b of a peer touch the SAME stage
// bytes whatever the alignment of their own `buf`; only the local side falls back to byte accesses when `buf` is not
// 16 B-aligned.
__global__ void __launch_bounds__(kThreads, 1)
    k_broadcast(CommDev c, uint8_t* buf, unsigned long long bytes, int root) {
  using namespace dev;
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  const bool aligned = (reinterpret_cast<uintptr_t>(buf) & 15u) == 0;
  const unsigned long long nvec = bytes / 16;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (c.rank == root) {
    for (unsigned long long v = first; v < nvec; v += stride) {
      uint4 q;
      if (aligned) {
        q = ldg_u4(buf + v * 16);
      } else {
        uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i >> 2] |= static_cast<uint32_t>(buf[v * 16 + i]) << ((i & 3) * 8);
        q = make_uint4(w[0], w[1], w[2], w[3]);
      }
#pragma unroll
      for (int jj = 1; jj < B2_MAX_WORLD; ++jj)
        if (jj < c.world) stg_u4(c.peer[jj] + stage + v * 16, q);
    }
    for (unsigned long long b = nvec * 16 + first; b < bytes; b += stride) {
      const uint8_t x = buf[b];
#pragma unroll
      for (int jj = 1; jj < B2_MAX_WORLD; ++jj)
        if (jj < c.world) c.peer[jj][stage + b] = x;
    }
  }
  cta_xbar(c, seq0 * 4u + 1u);
  if (c.rank != root) {
    const uint8_t* src = c.peer[0] + stage;
    for (unsigned long long v = first; v < nvec; v += stride) {
      const uint4 q = ldg_u4(src + v * 16);
      if (aligned) {
        stg_u4(buf + v * 16, q);
      } else {
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 16; ++i) buf[v * 16 + i] = static_cast<uint8_t>(w[i >> 2] >> ((i & 3) * 8));
      }
    }
    for (unsigned long long b = nvec * 16 + first; b < bytes; b += stride) buf[b] = src[b];
  }
  op_end(c);
}

__global__ void __launch_bounds__(kThreads, 1) k_barrier(CommDev c) {
  using namespace dev;
  const uint64_t seq0 = op_begin(c);
  cta_xbar(c, seq0 * 4u + 1u);
  op_end(c);
}
