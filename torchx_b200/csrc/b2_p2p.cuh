// b2_p2p.cuh — point-to-point send / recv (b2_p2p): a batch of sends and receives to and from any peers in ONE launch.
// A pure byte copy, like the all-to-all: every dtype is the same kernel.
//
// Channels.  A channel is an ordered pair (sender -> receiver); its messages match in issue order.  Each message is cut
// into chunks of at most kP2pPayload bytes (a 0-byte message is one header-only chunk), and chunk n of the channel's
// lifetime travels through slot n % kP2pSlots of the receiver's inbox for that sender.  Per slot, the chain is the flag
// barrier's (DESIGN.md 2.2):
//   sender   : ld.acquire.sys credit[slot] >= n + 1 - K (own arena) -> bar.sync -> header + data stores into the slot ->
//              bar.sync -> st.release.sys flag[slot] = n + 1 (receiver's arena)
//   receiver : ld.acquire.sys flag[slot] >= n + 1 (own arena) -> bar.sync -> header check, slot loads, stores to the
//              destination -> bar.sync -> st.release.sys credit[slot] = n + 1 (sender's arena)
// The credit's release orders the receiver's LOADS of the slot before the sender's next stores into it.
//
// Point-to-point never touches the collectives' state: not opseq / done, not the xbar or pipeline flags, not the stages or
// the LL buffers.  Its own device counters (chunks sent to / received from each peer, advanced by the last CTA of every
// launch) keep the host stateless, as opseq does for the collectives.
//
// Grid: the host gives every channel of the batch its own CTAs (at least one); a CTA never serves two channels.  A
// channel's chunks are striped over its CTAs and each CTA handles its chunks in increasing order, so the lowest unfinished
// chunk of every channel can always proceed: a send waits only on its own channel's older credits, a receive only on its
// own channel's data.  The two ends of a channel may run different grids: slots carry their own flags and credits.
#pragma once

#include "b2_dev.cuh"
#include "b2_exact.cuh"

namespace {

constexpr int kP2pSlots = 8;                          // K: slots per inbox (a power of two)
constexpr size_t kP2pSlotBytes = 512u << 10;          // one chunk: a 16-byte header + its payload
constexpr size_t kP2pHeaderBytes = 16;                // {byte count of the message lo, hi, 0, 0}
constexpr size_t kP2pPayload = kP2pSlotBytes - kP2pHeaderBytes;
constexpr size_t kP2pLineBytes = 128;                 // one flag or credit per 128-byte line
constexpr int kP2pLineWords = kP2pLineBytes / 4;
constexpr int kP2pMaxChans = 2 * (B2_MAX_WORLD - 1);  // (peer, direction) pairs
static_assert((kP2pSlots & (kP2pSlots - 1)) == 0, "kP2pSlots must be a power of two");

// Point-to-point region of an arena (after the LL buffers), for world W:
//   [ flags: (W-1) x K lines | credits: (W-1) x K lines | inboxes: (W-1) x K slots ]
// Inbox / flag block q of rank r belongs to sender s = q < r ? q : q + 1; credit block q of rank s to receiver
// r = q < s ? q : q + 1.
__host__ __device__ constexpr size_t p2p_lines_bytes(int world) {
  return static_cast<size_t>(world - 1) * kP2pSlots * kP2pLineBytes;
}
__host__ __device__ constexpr size_t p2p_region_bytes(int world) {
  return 2 * p2p_lines_bytes(world) + static_cast<size_t>(world - 1) * kP2pSlots * kP2pSlotBytes;
}

struct P2pChan {
  uint8_t* inbox;    // the K slots of this channel (receiver's arena)
  uint32_t* flag;    // K flag lines (receiver's arena)
  uint32_t* credit;  // K credit lines (sender's arena)
  uint32_t* count;   // this rank's device counter of the channel: chunks sent / received so far
  int cta_begin;     // first CTA of the channel; its CTAs run up to the next channel's cta_begin (or the grid's end)
  int send;          // this rank is the channel's sender
  uint32_t nchunks;  // chunks of this launch on the channel
};

struct P2pOp {
  uint8_t* ptr;
  unsigned long long bytes;
  uint32_t chan;    // index into P2pArgs::chan
  uint32_t chunk0;  // the op's first chunk, counted from the channel's first chunk of this launch
  uint32_t nchunks;
};

// One batch's kernel parameters (~2.8 KiB, by value: constant bank).
struct P2pArgs {
  P2pChan chan[kP2pMaxChans];
  P2pOp op[B2_P2P_MAX_OPS];
  int nchan;
  int nops;
  uint32_t* done;                  // CTAs of this launch that reached the end (own word, next to the channel counters)
  uint32_t* status;                // host-mapped: word 0 the B2_E* code, word 1 which kernel recorded B2_EINVAL
  unsigned long long timeout_ns;
};

constexpr uint32_t kStatusP2p = 1;  // status word 1: a byte-count mismatch of a receive

}  // namespace

namespace p2p {

// Bounded wait until *flag >= want (wrap-safe), as dev::wait_flag; false if it gave up.  A wait gives up after the
// communicator's timeout (recording B2_ETIMEOUT unless another code was recorded first), or as soon as it finds the
// status word already set: once one wait of this communicator has given up, or a receive has found a byte-count
// mismatch, every later wait stops within a few polls instead of spending a full timeout per chunk.  A wait that
// succeeds at once never reads the status word.
__device__ __forceinline__ bool wait(const P2pArgs& a, const uint32_t* flag, uint32_t want) {
  unsigned long long t0 = 0;
  unsigned spins = 0;
  while (static_cast<int32_t>(dev::ld_acquire_sys(flag) - want) < 0) {
    if ((++spins & 63u) == 0) {
      if (dev::ld_volatile_u32(a.status) != 0) return false;
      const unsigned long long now = dev::globaltimer_ns();
      if (t0 == 0) {
        t0 = now;
      } else if (now - t0 > a.timeout_ns) {
        dev::record_status(a.status, B2_ETIMEOUT);
        return false;
      }
    }
  }
  return true;
}

// Chunk j of `op`, chunk n of the channel's lifetime, into its slot of the receiver's inbox.  A sender whose credit wait
// gave up stores nothing and publishes nothing: the slot may still hold a chunk the receiver has not copied out, and a
// receiver that arrives late then waits for this chunk and records its own timeout instead of taking stale bytes.
__device__ __forceinline__ void send_chunk(const P2pArgs& a, const P2pChan& ch, const P2pOp& op, uint32_t j, uint32_t n) {
  const uint32_t slot = n & (kP2pSlots - 1);
  bool ok = true;
  if (threadIdx.x == 0) ok = wait(a, ch.credit + slot * kP2pLineWords, n + 1u - kP2pSlots);
  if (!__syncthreads_and(ok)) return;
  uint8_t* dst = ch.inbox + slot * kP2pSlotBytes;
  const unsigned long long off = static_cast<unsigned long long>(j) * kP2pPayload;
  const unsigned long long nb = op.bytes - off < kP2pPayload ? op.bytes - off : kP2pPayload;
  if (threadIdx.x == 0) dev::stg_u4(dst, make_uint4(static_cast<uint32_t>(op.bytes), static_cast<uint32_t>(op.bytes >> 32), 0u, 0u));
  const uint8_t* src = op.ptr + off;
  const bool aligned = (reinterpret_cast<uintptr_t>(src) & 15u) == 0;
  for (unsigned long long v = threadIdx.x; v < (nb + 15) / 16; v += kThreads)
    dev::stg_u4(dst + kP2pHeaderBytes + v * 16, exact::ld_local<1>(src, aligned, v, nb));
  __syncthreads();  // every thread's stores are ordered before the release below
  if (threadIdx.x == 0) dev::st_release_sys(ch.flag + slot * kP2pLineWords, n + 1u);
}

// Chunk j of `op` out of its slot of this rank's inbox.  A header whose byte count is not the op's: nothing is written,
// B2_EINVAL is recorded (unless a timeout was recorded first), and the slot is still handed back.  A receiver whose flag
// wait gave up writes nothing and hands nothing back.
__device__ __forceinline__ void recv_chunk(const P2pArgs& a, const P2pChan& ch, const P2pOp& op, uint32_t j, uint32_t n) {
  const uint32_t slot = n & (kP2pSlots - 1);
  bool ok = true;
  if (threadIdx.x == 0) ok = wait(a, ch.flag + slot * kP2pLineWords, n + 1u);
  if (!__syncthreads_and(ok)) return;  // the sender's stores are now visible to every thread of this CTA
  const uint8_t* src = ch.inbox + slot * kP2pSlotBytes;
  const uint4 h = dev::ldg_u4(src);
  if (((static_cast<unsigned long long>(h.y) << 32) | h.x) == op.bytes) {
    const unsigned long long off = static_cast<unsigned long long>(j) * kP2pPayload;
    const unsigned long long nb = op.bytes - off < kP2pPayload ? op.bytes - off : kP2pPayload;
    uint8_t* dst = op.ptr + off;
    const bool aligned = (reinterpret_cast<uintptr_t>(dst) & 15u) == 0;
    for (unsigned long long v = threadIdx.x; v < (nb + 15) / 16; v += kThreads)
      exact::st_local<1>(dst, aligned, v, nb, dev::ldg_u4(src + kP2pHeaderBytes + v * 16));
  } else if (threadIdx.x == 0 && dev::ld_volatile_u32(a.status) == 0) {
    reinterpret_cast<volatile uint32_t*>(a.status)[1] = kStatusP2p;
    __threadfence_system();
    dev::record_status(a.status, B2_EINVAL);
  }
  __syncthreads();  // every thread's loads of the slot are ordered before the release below
  if (threadIdx.x == 0) dev::st_release_sys(ch.credit + slot * kP2pLineWords, n + 1u);
}

}  // namespace p2p

__global__ void __launch_bounds__(kThreads, 1) k_p2p(P2pArgs a) {
  int c = 0;
  for (int i = 1; i < a.nchan; ++i)
    if (static_cast<int>(blockIdx.x) >= a.chan[i].cta_begin) c = i;
  const P2pChan ch = a.chan[c];
  const uint32_t G = static_cast<uint32_t>((c + 1 < a.nchan ? a.chan[c + 1].cta_begin : static_cast<int>(gridDim.x)) - ch.cta_begin);
  const uint32_t k = blockIdx.x - ch.cta_begin;
  const uint32_t n0 = dev::ld_volatile_u32(ch.count);
  for (int o = 0; o < a.nops; ++o) {
    if (a.op[o].chan != static_cast<uint32_t>(c)) continue;
    const P2pOp op = a.op[o];
    for (uint32_t j = (k + G - op.chunk0 % G) % G; j < op.nchunks; j += G) {
      if (ch.send) p2p::send_chunk(a, ch, op, j, n0 + op.chunk0 + j);
      else p2p::recv_chunk(a, ch, op, j, n0 + op.chunk0 + j);
    }
  }
  // the last CTA advances every channel's counter (every CTA has read its n0 by then), as op_end does opseq
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(a.done, 1u) == gridDim.x - 1) {
      for (int i = 0; i < a.nchan; ++i) *reinterpret_cast<volatile uint32_t*>(a.chan[i].count) = dev::ld_volatile_u32(a.chan[i].count) + a.chan[i].nchunks;
      *reinterpret_cast<volatile uint32_t*>(a.done) = 0;
      __threadfence();
    }
  }
}
