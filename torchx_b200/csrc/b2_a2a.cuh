// b2_a2a.cuh — all-to-all (b2_alltoall): rank r's block j goes to rank j and lands in rank j's r-th output, with any byte
// count per (sender, receiver) pair, in ONE launch per call.  A pure byte copy: every dtype and layout is the same kernel.
//   A  push : send[jj] -> recv[me] of rank (me + jj) % W, behind a 16-byte header {count lo, count hi, abort, 0}
//   B  copy : if no header carries the abort flag and every count is what this rank expects, copy recv[r] of the own stage
//             out to its destination, and the own block straight from send[0] to recv[0]
// One cta_xbar between them.
//
// No rank knows the other ranks' counts, so:
//   * the grid depends only on W, the stage size and max_ctas (the host sizes it for the per-pair capacity).  cta_xbar pairs
//     CTAs with equal blockIdx.x across ranks, and when the counts agree the CTA that copies vec v of region r out in phase B
//     is the one whose partner on rank r pushed it;
//   * thread 0 of EVERY CTA writes the headers: a CTA is only ordered after the CTAs of its own index on the other ranks, so
//     a header written by CTA 0 alone could still be in flight when CTA b reads it.  Every CTA reads the same headers and
//     makes the same decision;
//   * a disagreement cannot be resolved inside the kernel.  A pair over the per-pair limit is seen on the host by both its
//     ranks, which launch with `abort` set: they push no data and the abort flag reaches every rank after the one barrier.
//     A count that differs from what this rank expects (the own pair's two counts included) is seen only here.  Either way
//     this rank writes none of its outputs and records B2_EINVAL in the host-mapped status word (b2_comm_status).
// The op counter, stage parity and flag sequence are those of every other collective.
#pragma once

#include "b2_dev.cuh"
#include "b2_exact.cuh"

namespace {

// One all-to-all's kernel parameters, rotated like CommDev::peer: entry jj belongs to rank (rank + jj) % world, so the
// unrolled loops read them with compile-time indices (constant bank) and never from a local-memory copy.
struct A2aArgs {
  const uint8_t* send[B2_MAX_WORLD];            // what goes to that rank (may be null when its count is 0)
  unsigned long long send_bytes[B2_MAX_WORLD];
  uint8_t* recv[B2_MAX_WORLD];                  // where that rank's bytes land (may be null when its count is 0)
  unsigned long long recv_bytes[B2_MAX_WORLD];
  uint32_t abort;                               // nonzero: push no data, make every rank give up the exchange
};

constexpr size_t kA2aHeaderBytes = 16;  // at the start of every recv region; a pair carries at most slice_cap - 16 bytes

}  // namespace

__global__ void __launch_bounds__(kThreads, 1) k_alltoall(CommDev c, A2aArgs a) {
  using namespace dev;
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;

  // ---- phase A: header and data into recv[me] of every peer --------------------------------------------
#pragma unroll
  for (int jj = 1; jj < B2_MAX_WORLD; ++jj) {
    if (jj < c.world) {
      uint8_t* dst = c.peer[jj] + stage + c.rank * c.slice_cap;
      const unsigned long long count = a.send_bytes[jj];
      if (threadIdx.x == 0)
        stg_u4(dst, make_uint4(static_cast<uint32_t>(count), static_cast<uint32_t>(count >> 32), a.abort, 0u));
      const unsigned long long n = a.abort ? 0ull : count;
      const uint8_t* src = a.send[jj];
      const bool aligned = (reinterpret_cast<uintptr_t>(src) & 15u) == 0;
      for (unsigned long long v = first; v < (n + 15) / 16; v += stride)
        stg_u4(dst + kA2aHeaderBytes + v * 16, exact::ld_local<1>(src, aligned, v, n));
    }
  }
  cta_xbar(c, seq0 * 4u + 1u);

  // ---- phase B: check the headers, then copy every region out --------------------------------------------
  const uint8_t* mine = c.peer[0] + stage;
  bool ok = a.abort == 0 && a.send_bytes[0] == a.recv_bytes[0];
#pragma unroll
  for (int jj = 1; jj < B2_MAX_WORLD; ++jj) {
    if (jj < c.world) {
      const uint4 h = ldg_u4(mine + rank_at(c, jj) * c.slice_cap);  // the header of rank (rank + jj) % world
      const unsigned long long count = (static_cast<unsigned long long>(h.y) << 32) | h.x;
      ok = ok && h.z == 0 && count == a.recv_bytes[jj];
    }
  }
  if (ok) {
#pragma unroll
    for (int jj = 0; jj < B2_MAX_WORLD; ++jj) {
      if (jj < c.world) {
        const int r = rank_at(c, jj);
        const unsigned long long n = a.recv_bytes[jj];
        uint8_t* dst = a.recv[jj];
        const bool dst_aligned = (reinterpret_cast<uintptr_t>(dst) & 15u) == 0;
        const bool src_aligned = (reinterpret_cast<uintptr_t>(a.send[0]) & 15u) == 0;
        const uint8_t* region = mine + r * c.slice_cap + kA2aHeaderBytes;  // whole vecs, 16 B-aligned
        for (unsigned long long v = first; v < (n + 15) / 16; v += stride) {
          const uint4 q = jj == 0 ? exact::ld_local<1>(a.send[0], src_aligned, v, n) : ldg_u4(region + v * 16);
          exact::st_local<1>(dst, dst_aligned, v, n, q);
        }
      }
    }
  } else if (blockIdx.x == 0 && threadIdx.x == 0 && ld_volatile_u32(c.status) == 0) {  // a timeout recorded first stays
    record_status(c.status, B2_EINVAL);
  }
  op_end(c);
}
