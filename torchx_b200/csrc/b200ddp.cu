// b200ddp.cu — libb200ddp.so: H100 (sm_90a) data plane for the `local_cuda` TorchX scheduler.
//
// What lives here (see include/b200ddp.h for the ABI and DESIGN.md for the rationale):
//   * rendezvous: POSIX-shm control block + exchange of ONE symmetric arena per rank, either as CUDA VMM allocations
//     shared by file descriptor and bound into an NVSwitch MULTICAST object (b2_vmm.h), or - when the driver / fabric
//     does not offer that - as cudaMalloc + CUDA IPC
//     (replaces c10d TCPStore + ncclCommInitRank on the reference path,
//      torchx/distributed/__init__.py:217-222 -> torch.distributed.init_process_group)
//   * the DDP gradient-bucket allreduce as ONE fused kernel per bucket
//     (replaces the 4-launch cast -> div -> ncclAllReduce -> copy sequence of
//      torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py:57-93)
//       - one-shot        : push compressed message to every peer, one flag barrier, reduce locally   (b2_kernels.cuh)
//       - two-shot        : push-scatter -> reduce own slice -> pull-gather, single pass              (b2_kernels.cuh)
//       - two-shot, piped : the same three phases as warp-specialised roles over K chunks            (b2_pipe.cuh)
//       - NVLS, piped     : cast -> multimem.ld_reduce / multimem.st through the switch -> widen      (b2_pipe.cuh)
//   * broadcast / barrier on the same fabric (DDP init + BN-buffer sync, dist.barrier()).
//   * the exact collectives of a training script: integer SUM and MIN / MAX allreduce, all-gather (b2_exact.cuh).
//   * reduce-scatter with the allreduce's arithmetic: push-scatter, one barrier, reduce own block (b2_rs.cuh).
//   * reduce to a root: the reduce-scatter's reduced slices pulled by the root alone (b2_reduce.cuh).
//   * all-to-all with any split sizes: push each block behind a count header, one barrier, copy out (b2_a2a.cuh).
//   * point-to-point send / recv in batches: per-channel slot inboxes with flags and credits, no barrier (b2_p2p.cuh).
//   * SyncBatchNorm's statistics exchange: gather + merge of every rank's mean / invstd / count (b2_bnstats.cuh).
//   * the elementwise passes of training-mode BatchNorm2d on channels-last bf16 activations (b2_bn.cuh).
//
// Memory model: every cross-GPU hand-off is  data stores -> bar.sync -> st.release.sys(flag)
// on the producer and  ld.acquire.sys(flag) -> bar.sync -> data loads  on the consumer, with a
// monotonically increasing sequence number instead of flag resets (no ABA, no reset races).
// All peer waits are bounded: a CTA that waits longer than `timeout_ns` records B2_ETIMEOUT in a
// host-mapped status word and carries on, so a dead peer can never hang the GPU.
//
// No tensor cores: the path is a pure bandwidth-bound reduction (1 add per 2-4 bytes moved).

#include "b2_dev.cuh"
#include "b2_kernels.cuh"
#include "b2_pipe.cuh"
#include "b2_ll.cuh"
#include "b2_exact.cuh"
#include "b2_rs.cuh"
#include "b2_reduce.cuh"
#include "b2_a2a.cuh"
#include "b2_p2p.cuh"
#include "b2_bnstats.cuh"
#include "b2_bn.cuh"
#include "b2_vmm.h"

#include <errno.h>
#include <fcntl.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <atomic>
#include <map>
#include <mutex>
#include <new>
#include <string>

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
  char tmp[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tmp, sizeof(tmp), fmt, ap);
  va_end(ap);
  g_err = tmp;
  return code;
}

#define B2_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t e__ = (expr);                                                                 \
    if (e__ != cudaSuccess)                                                                   \
      return fail(B2_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, \
                  __LINE__);                                                                  \
  } while (0)

struct DeviceGuard {  // the library never leaves the caller's current device changed
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

double now_s() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

// ---- shm control block (multi-process rendezvous) ----------------------------------------------
constexpr uint64_t kShmMagic = 0x42323030444451ull;  // "B200DDQ": layout 2

struct ShmSlot {
  cudaIpcMemHandle_t handle;  // cudaMalloc backend only
  int device;        // the rank's ordinal in ITS OWN numbering (CUDA_VISIBLE_DEVICES may differ between ranks)
  char bus_id[24];   // PCI bus id: the identity that is comparable across processes
  int pid;
  int cap_vmm;       // this rank can build its arena from VMM objects and pass file descriptors
  int cap_mc;        // ... and its device supports NVSwitch multicast
  unsigned long long arena_bytes;
  std::atomic<uint32_t> hello;  // 1 once cap_* are valid (backend agreement happens before any allocation)
  std::atomic<uint32_t> ready;  // 1 once handle/device/pid/arena_bytes are valid and the fd socket is bound
  char pad[64];
};

struct ShmBlock {
  std::atomic<uint64_t> magic;
  uint64_t epoch;
  int world;
  std::atomic<int> mapped;     // ranks that have mapped every peer arena
  std::atomic<int> departed;   // ranks that have finished using peer memory (destroy handshake)
  std::atomic<int> mc_added;   // multicast: ranks past cuMulticastAddDevice
  std::atomic<int> mc_bound;   // ... past cuMulticastBindMem
  std::atomic<int> mc_mapped;  // ... past mapping the multicast object
  std::atomic<int> mc_fail;    // any rank failed a multicast step: everybody drops the NVLS path
  ShmSlot slot[B2_MAX_WORLD];
};

// the multicast mapping of an in-process world is shared by its ranks
struct LocalMc {
  vmm::Mapping map;
  int refs = 0;
};

// What B2_ALGO_AUTO picks (auto_algo), in wire bytes of the message.
struct AutoPolicy {
  size_t oneshot_max;  // one-shot up to this many
  size_t ll_min;       // the barrier-free LL two-shot from this many (above the one-shot range) ...
  size_t ll_max;       // ... up to (excluding) this many
  size_t pipe_min;     // the pipelined kernels from this many
  size_t nvls_min;     // NVLS (when available and the mode allows it) from this many ...
  int nvls_min_world;  // ... and this world size: NVLS only pays once (1 + 1/W) < 2 (W-1)/W
};

}  // namespace

struct b2_comm {
  CommDev d{};
  int device = -1;
  bool local_world = false;    // created by b2_comm_create_local (no IPC, no shm)
  bool use_vmm = false;        // arena built from VMM objects (else cudaMalloc [+ CUDA IPC])
  bool peer_is_ipc[B2_MAX_WORLD] = {};
  uint8_t* arena_of[B2_MAX_WORLD] = {};  // arena_of[r] = rank r's arena as mapped in this process
  void* arena = nullptr;       // this rank's arena: [xbar flags | pipeline flags | stage0 | stage1 | LL0 | LL1 | p2p]
  size_t arena_bytes = 0;
  size_t stage_bytes = 0;
  vmm::Mapping own;                  // VMM backend: my physical allocation + its mapping
  vmm::Mapping peers[B2_MAX_WORLD];  // VMM backend, multi-process: imported peer allocations
  vmm::Mapping mc;                   // VMM backend, multi-process: the multicast object
  LocalMc* local_mc = nullptr;       // VMM backend, in-process world
  uint32_t* counters = nullptr;  // cudaMalloc'ed, 256 B: opseq (u64, words 0-1), done (word 32)
  uint32_t* p2p_counters = nullptr;  // cudaMalloc'ed: chunks sent to [0, W) / received from [8, 8 + W) each rank; [32] done
  size_t p2p_off = 0;                // the point-to-point region of every arena (b2_p2p.cuh)
  unsigned long long* trace_dev = nullptr;  // cudaMalloc'ed on demand: kMaxCtas * 8 stamps
  uint32_t* status_host = nullptr;
  // tuning (identical on every rank: they come from the same environment / the same b2_comm_set_param calls)
  int max_ctas = 0;                 // 0 = heuristic
  AutoPolicy policy{};
  size_t pipe_chunk_bytes = 0;        // target wire bytes of one pipeline chunk (per rank)
  uint64_t launches = 0;
  int last_algo = 0;                  // B2_ALGO_* of the most recent allreduce launch (what AUTO picked)
  ShmBlock* shm = nullptr;
  std::string shm_path;
};

namespace {

size_t env_size(const char* name, size_t dflt) {
  const char* s = getenv(name);
  if (!s || !*s) return dflt;
  char* end = nullptr;
  unsigned long long v = strtoull(s, &end, 10);
  return end == s ? dflt : static_cast<size_t>(v);
}

// Largest message (in wire bytes) for which AUTO takes one-shot: one-shot moves (W-1)x the payload per rank but needs
// one barrier instead of two, so the crossover falls quickly with W.  At W=2 both move the same bytes and one-shot wins
// until HBM traffic dominates.
size_t default_oneshot_max(int world) {
  if (world <= 2) return 16u << 20;
  if (world <= 4) return 2u << 20;
  return 512u << 10;
}

AutoPolicy default_policy(int world) {
  AutoPolicy p;
  p.oneshot_max = env_size("B2_ONESHOT_MAX_BYTES", default_oneshot_max(world));
  p.pipe_min = env_size("B2_PIPE_MIN_BYTES", ~static_cast<size_t>(0));
  p.nvls_min = env_size("B2_NVLS_MIN_BYTES", 64u << 20);
  p.nvls_min_world = static_cast<int>(env_size("B2_NVLS_MIN_WORLD", 8));
  p.ll_min = env_size("B2_LL_MIN_BYTES", world >= 3 ? 0 : ~static_cast<size_t>(0));
  p.ll_max = env_size("B2_LL_MAX_BYTES", 8u << 20);
  return p;
}

// What B2_ALGO_AUTO resolves to for one launch (DESIGN.md 2.6).  Pure: the same inputs give the same answer on every rank.
int auto_algo(const AutoPolicy& p, int world, int mode, size_t wire_bytes, bool multicast, bool fits_oneshot) {
  // fp32-wire NVLS would let the switch pick the fp32 summation order; AUTO keeps that mode on the rank-order kernels
  if (multicast && mode != B2_F32 && world >= p.nvls_min_world && wire_bytes >= p.nvls_min) return B2_ALGO_NVLS;
  if (wire_bytes <= p.oneshot_max && fits_oneshot) return B2_ALGO_ONESHOT;
  if (wire_bytes >= p.ll_min && wire_bytes < p.ll_max) return B2_ALGO_TWOSHOT_LL;
  if (wire_bytes >= p.pipe_min) return B2_ALGO_TWOSHOT_PIPE;
  return B2_ALGO_TWOSHOT;
}

// Arena layout for a given world size; fills d.*_off / d.slice_cap and arena_bytes (before backend rounding).
void layout(b2_comm* c, int world, size_t stage_bytes) {
  size_t cap = stage_bytes / (world + 1);
  cap &= ~static_cast<size_t>(255);
  c->stage_bytes = cap * (world + 1);
  c->d.slice_cap = cap;
  c->d.flag_off = 0;
  c->d.pflag_off = kXbarFlagBytes;
  c->d.stage_off[0] = kFlagRegionBytes;
  c->d.stage_off[1] = kFlagRegionBytes + c->stage_bytes;
  c->arena_bytes = kFlagRegionBytes + 2 * c->stage_bytes;
  // the sentinel-managed buffers (LL two-shot recv/out, NVLS out): 2W regions per parity
  const size_t ll_bytes = 2 * static_cast<size_t>(world) * cap;
  c->d.ll_off[0] = c->arena_bytes;
  c->d.ll_off[1] = c->arena_bytes + ll_bytes;
  c->arena_bytes += 2 * ll_bytes;
  c->d.llflag_off = kLLFlagOff;
  // point-to-point inboxes, flags and credits: after everything the collectives use, a function of the world size alone
  c->p2p_off = c->arena_bytes;
  c->arena_bytes += p2p_region_bytes(world);
}

// Everything of a rank except the arena itself.
int init_rank(b2_comm* c, int rank, int world, int device, size_t stage_bytes) {
  c->device = device;
  c->d.rank = rank;
  c->d.world = world;
  if (stage_bytes == 0) stage_bytes = env_size("B2_STAGE_MB", kDefaultStageBytes >> 20) << 20;
  if (stage_bytes < (static_cast<size_t>(world + 1) << 12))
    return fail(B2_EINVAL, "stage_bytes=%zu too small for world=%d", stage_bytes, world);
  c->d.timeout_ns = env_size("B2_TIMEOUT_MS", kDefaultTimeoutNs / 1000000ull) * 1000000ull;
  layout(c, world, stage_bytes);
  c->max_ctas = static_cast<int>(env_size("B2_MAX_CTAS", 0));
  // AUTO thresholds, in wire bytes (every one can be moved with an environment variable or b2_comm_set_param):
  //   one-shot            up to default_oneshot_max(world)
  //   LL two-shot         from there to 8 MiB at W >= 3 (at W=2 one-shot covers that range: off)
  //   single-pass two-shot  above that (the DDP 25 MiB buckets: the kernel with no extra local traffic when backward
  //                       competes for HBM inside the training step)
  //   NVLS                from 64 MiB at W = 8; the switch's arithmetic, within one bf16 ulp of the exact sum (DESIGN.md 2.4)
  //   pipelined two-shot  never (explicit choice only)
  // The crossovers have not been re-measured on multi-GPU H100 systems.
  c->policy = default_policy(world);
  c->pipe_chunk_bytes = env_size("B2_PIPE_CHUNK_KB", 2048) << 10;
  B2_CUDA(cudaSetDevice(device));
  B2_CUDA(cudaMalloc(&c->counters, 256));
  B2_CUDA(cudaMemset(c->counters, 0, 256));
  c->d.opseq = reinterpret_cast<uint64_t*>(c->counters);
  c->d.done = c->counters + 32;  // a different 128 B line
  B2_CUDA(cudaMalloc(&c->p2p_counters, 256));
  B2_CUDA(cudaMemset(c->p2p_counters, 0, 256));
  B2_CUDA(cudaHostAlloc(&c->status_host, 64, cudaHostAllocMapped | cudaHostAllocPortable));
  memset(c->status_host, 0, 64);
  void* sdev = nullptr;
  B2_CUDA(cudaHostGetDevicePointer(&sdev, c->status_host, 0));
  c->d.status = static_cast<uint32_t*>(sdev);
  return B2_OK;
}

// This rank's arena.  VMM backend: a shareable physical allocation mapped for `devices` (the rank's own device in the
// one-process-per-GPU case, every device of the world for an in-process world).  Legacy backend: cudaMalloc.
int alloc_arena(b2_comm* c, bool use_vmm, bool multicast, const int* devices, int ndev) {
  B2_CUDA(cudaSetDevice(c->device));
  c->use_vmm = use_vmm;
  if (use_vmm) {
    const size_t gran = vmm::arena_granularity(c->device, c->d.world, multicast);
    c->arena_bytes = (c->arena_bytes + gran - 1) / gran * gran;
    const CUmemAllocationProp prop = vmm::alloc_prop(c->device);
    const CUresult r = vmm::driver().MemCreate(&c->own.handle, c->arena_bytes, &prop, 0);
    if (r != CUDA_SUCCESS) return fail(B2_ECUDA, "cuMemCreate(%zu bytes): %s", c->arena_bytes, vmm::errstr(r).c_str());
    const std::string e = vmm::map_handle(&c->own, c->arena_bytes, gran, devices, ndev);
    if (!e.empty()) return fail(B2_ECUDA, "mapping this rank's arena: %s", e.c_str());
    c->arena = reinterpret_cast<void*>(c->own.va);
  } else {
    B2_CUDA(cudaMalloc(&c->arena, c->arena_bytes));
  }
  B2_CUDA(cudaMemset(c->arena, 0, kFlagRegionBytes));
  B2_CUDA(cudaMemset(static_cast<uint8_t*>(c->arena) + c->d.ll_off[0], 0xFF, 4 * static_cast<size_t>(c->d.world) * c->d.slice_cap));
  B2_CUDA(cudaMemset(static_cast<uint8_t*>(c->arena) + c->p2p_off, 0, 2 * p2p_lines_bytes(c->d.world)));  // flags and credits
  B2_CUDA(cudaDeviceSynchronize());
  c->arena_of[c->d.rank] = static_cast<uint8_t*>(c->arena);
  return B2_OK;
}

void rotate_peers(b2_comm* c) {
  for (int jj = 0; jj < c->d.world; ++jj) c->d.peer[jj] = c->arena_of[(c->d.rank + jj) % c->d.world];
}

void free_rank_resources(b2_comm* c) {
  if (c->device >= 0) cudaSetDevice(c->device);
  if (c->use_vmm) {
    if (c->local_mc && --c->local_mc->refs == 0) {
      vmm::unmap_release(&c->local_mc->map);
      delete c->local_mc;
    }
    c->local_mc = nullptr;
    vmm::unmap_release(&c->mc);
    for (int r = 0; r < B2_MAX_WORLD; ++r) vmm::unmap_release(&c->peers[r]);
    vmm::unmap_release(&c->own);
  } else if (c->arena) {
    cudaFree(c->arena);
  }
  if (c->counters) cudaFree(c->counters);
  if (c->p2p_counters) cudaFree(c->p2p_counters);
  if (c->trace_dev) cudaFree(c->trace_dev);
  c->trace_dev = nullptr;
  if (c->status_host) cudaFreeHost(c->status_host);
  c->arena = nullptr;
  c->counters = nullptr;
  c->p2p_counters = nullptr;
  c->status_host = nullptr;
}

int grid_for(const b2_comm* c, unsigned long long vecs_per_cta_dim, int unroll) {
  // Enough CTAs that each thread has work, capped so the collective leaves SMs to the backward
  // pass it overlaps with.  Deterministic in (n, world, max_ctas) => identical on every rank.
  // Default cap: 64 CTAs; 128 once 64 CTAs would each loop more than twice (from ~16 MiB fp32 buckets at W=8).  One CTA
  // per SM (512 threads, <= 128 regs), so even the larger grid stays within the 132 SMs of an H100.
  const int dflt = vecs_per_cta_dim > 64ull * kThreads * static_cast<unsigned long long>(unroll) * 2ull ? 128 : 64;
  const int cap = c->max_ctas > 0 ? (c->max_ctas > kMaxCtas ? kMaxCtas : c->max_ctas) : dflt;
  unsigned long long per = static_cast<unsigned long long>(kThreads) * unroll;
  unsigned long long g = (vecs_per_cta_dim + per - 1) / per;
  if (g < 1) g = 1;
  if (g > static_cast<unsigned long long>(cap)) g = cap;
  return static_cast<int>(g);
}

// SMs of `device` (132 on an H100 SXM, 114 on the PCIe card): the occupancy-sized grids of the local pass scale with it.
int sm_count(int device) {
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n < 1) {
    cudaGetLastError();
    n = 132;
  }
  return n;
}

// Pipelined kernels: grid g, K chunks, cell = vecs of one (chunk, CTA) cell of a slice (multiple of 32, so every warp
// access is a whole 512 B line group).  Deterministic in (Ls, wire bytes, tuning) => identical on every rank.
struct PipePlan {
  int grid;
  int K;
  unsigned long long cell;
};

PipePlan plan_pipe(const b2_comm* c, unsigned long long Ls, size_t wire_bytes) {
  const unsigned long long units = (Ls + 31) / 32;  // 32-vec units in a slice
  const int cap = c->max_ctas > 0 ? (c->max_ctas > kMaxCtas ? kMaxCtas : c->max_ctas)
                                  : (wire_bytes >= (8u << 20) ? 128 : 64);
  unsigned long long g = units < static_cast<unsigned long long>(cap) ? units : cap;
  if (g < 1) g = 1;
  unsigned long long K = c->pipe_chunk_bytes ? (wire_bytes + c->pipe_chunk_bytes / 2) / c->pipe_chunk_bytes : 1;
  if (K < 1) K = 1;
  if (K > static_cast<unsigned long long>(kMaxChunks)) K = kMaxChunks;
  const unsigned long long per_cta_units = (units + g - 1) / g;
  if (K > per_cta_units) K = per_cta_units;
  const unsigned long long cell_units = (units + g * K - 1) / (g * K);
  PipePlan p;
  p.grid = static_cast<int>(g);
  p.K = static_cast<int>(K);
  p.cell = cell_units * 32;
  return p;
}

// The world sizes of the multi-rank kernels: calls f(std::integral_constant<int, W>{}) and returns true for
// W = world in 2 .. B2_MAX_WORLD, or returns false.  Every runtime world size becomes a compile-time one here.
template <int W = 2, class F>
bool with_world(int world, F&& f) {
  if constexpr (W > B2_MAX_WORLD) {
    return false;
  } else {
    if (world != W) return with_world<W + 1>(world, f);
    f(std::integral_constant<int, W>{});
    return true;
  }
}

// One collective of `kind` (B2_ALGO_ONESHOT / TWOSHOT / TWOSHOT_PIPE / TWOSHOT_LL / NVLS) at the communicator's world size.
template <int MODE>
cudaError_t launch_collective(const CommDev& d, const Src& src, int kind, int grid, const PipePlan& p, void* buf,
                              unsigned long long n, float scale, cudaStream_t s) {
  cudaError_t e = cudaErrorInvalidValue;
  with_world(d.world, [&](auto w) {
    constexpr int W = decltype(w)::value;
    switch (kind) {
      case B2_ALGO_ONESHOT:
        k_oneshot<MODE, W><<<grid, kThreads, 0, s>>>(d, src, buf, n, scale);
        break;
      case B2_ALGO_TWOSHOT:
        k_twoshot<MODE, W><<<grid, kThreads, 0, s>>>(d, src, buf, n, scale);
        break;
      case B2_ALGO_TWOSHOT_PIPE:
        k_pipe<MODE, W, pl::kP2p><<<p.grid, kThreads, 0, s>>>(d, src, buf, n, scale, p.K, p.cell);
        break;
      case B2_ALGO_TWOSHOT_LL:
        k_ll<MODE, W><<<grid, kThreads, 0, s>>>(d, src, buf, n, scale);
        break;
      default:  // B2_ALGO_NVLS
        k_pipe<MODE, W, pl::kNvls><<<p.grid, kThreads, 0, s>>>(d, src, buf, n, scale, p.K, p.cell);
    }
    e = cudaGetLastError();
  });
  return e;
}

// The float reduce-scatter at the communicator's world size.
template <int MODE>
cudaError_t launch_reduce_scatter(const CommDev& d, const Src& src, int grid, void* out, const void* in, unsigned long long n,
                                  unsigned long long block, float scale, cudaStream_t s) {
  cudaError_t e = cudaErrorInvalidValue;
  with_world(d.world, [&](auto w) {
    k_reduce_scatter<MODE, decltype(w)::value><<<grid, kThreads, 0, s>>>(d, src, out, in, n, block, scale);
    e = cudaGetLastError();
  });
  return e;
}

// The local pass's grid over n elements: enough CTAs for 4 vecs per thread, at most 4 resident CTAs per SM (~64 KiB of
// loads in flight per SM).
int local_grid(unsigned long long n, unsigned long long sms) {
  const unsigned long long V = (n + 7) / 8;
  unsigned long long g = (V + kThreads * 4ull - 1) / (kThreads * 4ull);
  if (g < 1) g = 1;
  if (g > sms * 4) g = sms * 4;
  return static_cast<int>(g);
}

template <int MODE>
cudaError_t launch_local(const Src& src, void* buf, unsigned long long n, float scale, cudaStream_t s) {
  // TMA-staged path for 16 B-aligned buckets.  The ring needs several tiles per CTA to pay for its prologue, so it is
  // the default only for very large buckets (from 256 MiB up; a threshold not re-measured on H100).
  // B2_LOCAL_TMA_MIN_MB moves the threshold (0 = always for >= 1 MiB, e.g. for the parity tests), B2_LOCAL_TMA=0
  // disables it.
  static const bool use_tma = env_size("B2_LOCAL_TMA", 1) != 0;
  static const unsigned long long tma_min = env_size("B2_LOCAL_TMA_MIN_MB", 256) << 20;
  const unsigned long long nbytes = n * ModeTraits<MODE>::kElemBytes;
  int devno = 0;
  cudaGetDevice(&devno);
  const unsigned long long sms = static_cast<unsigned long long>(sm_count(devno));
  if (use_tma && src.nseg == 0 && (reinterpret_cast<uintptr_t>(buf) & 15u) == 0 && nbytes >= (1ull << 20) && nbytes >= tma_min) {
    const unsigned long long ntiles = nbytes / tma::kTileBytes;
    unsigned long long g = ntiles < sms * 2 ? ntiles : sms * 2;  // persistent: 2 CTAs (2 x 64 KiB rings) per SM
    constexpr int kSmem = tma::kStages * tma::kTileBytes;
    static std::atomic<unsigned> configured{0};  // bit d: the 64 KiB opt-in has been set on device d
    if (!(configured.load(std::memory_order_relaxed) & (1u << (devno & 31)))) {
      const cudaError_t attr = cudaFuncSetAttribute(k_local_pass_tma<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
      if (attr != cudaSuccess) return attr;
      configured.fetch_or(1u << (devno & 31), std::memory_order_relaxed);
    }
    k_local_pass_tma<MODE><<<static_cast<int>(g), tma::kTmaThreads, kSmem, s>>>(buf, n, scale);
    return cudaGetLastError();
  }
  k_local_pass<MODE><<<local_grid(n, sms), kThreads, 0, s>>>(src, buf, n, scale);
  return cudaGetLastError();
}

// The B2_* modes of include/b200ddp.h: calls f(std::integral_constant<int, MODE>{}) and returns true, or returns false
// for an unknown mode.  Every runtime mode becomes a compile-time one here, so a new mode is one more case.
template <class F>
bool with_mode(int mode, F&& f) {
  switch (mode) {
    case B2_F32_WIRE_BF16:
      f(std::integral_constant<int, B2_F32_WIRE_BF16>{});
      return true;
    case B2_F32:
      f(std::integral_constant<int, B2_F32>{});
      return true;
    case B2_BF16:
      f(std::integral_constant<int, B2_BF16>{});
      return true;
    case B2_F32_WIRE_F16:
      f(std::integral_constant<int, B2_F32_WIRE_F16>{});
      return true;
    case B2_F16:
      f(std::integral_constant<int, B2_F16>{});
      return true;
    default:
      return false;
  }
}

bool known_mode(int mode) {
  return with_mode(mode, [](auto) {});
}

size_t elem_bytes(int mode) {
  size_t b = 0;
  with_mode(mode, [&](auto m) { b = ModeTraits<decltype(m)::value>::kElemBytes; });
  return b;
}

size_t wire_vec_bytes(int mode) {
  size_t b = 0;
  with_mode(mode, [&](auto m) { b = dev::Wire<decltype(m)::value>::kBytes; });
  return b;
}

const Src kNoSrc = {};  // nseg == 0: the collective reads the bucket itself

// Calls launch(off, n) for the consecutive chunks [off, off + n) of [0, total), each of at most cap units, and counts each
// launch on c.  launch returns its launch error; the first failure ends the loop and is returned.
template <class F>
cudaError_t for_chunks(b2_comm* c, size_t total, size_t cap, F&& launch) {
  for (size_t off = 0; off < total;) {
    const size_t n = total - off < cap ? total - off : cap;
    const cudaError_t e = launch(off, n);
    if (e != cudaSuccess) return e;
    c->launches++;
    off += n;
  }
  return cudaSuccess;
}

// [p, p + n) and [q, q + m) share a byte (an empty range shares none).
bool overlaps(const void* p, size_t n, const void* q, size_t m) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
  return n && m && a < b + m && b < a + n;
}

int local_pass_impl(const Src& src, void* buf, size_t n_elems, int mode, float scale, int device, void* stream) {
  if (n_elems == 0) return B2_OK;
  if (!buf) return fail(B2_EINVAL, "b2_local_pass: null buffer");
  DeviceGuard g(device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (!with_mode(mode, [&](auto m) { e = launch_local<decltype(m)::value>(src, buf, n_elems, scale, s); }))
    return fail(B2_EINVAL, "unknown mode %d", mode);
  if (e != cudaSuccess) return fail(B2_ECUDA, "k_local_pass launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

unsigned next_creation_index(const char* shm_name, uint64_t epoch) {
  static std::mutex mu;
  static std::map<std::string, unsigned> seen;
  std::lock_guard<std::mutex> lock(mu);
  return seen[std::string(shm_name) + "#" + std::to_string(epoch)]++;
}

bool wait_count(std::atomic<int>& ctr, int target, std::atomic<int>* abort_flag, double deadline) {
  while (ctr.load(std::memory_order_acquire) < target) {
    if (abort_flag && abort_flag->load(std::memory_order_acquire)) return false;
    if (now_s() > deadline) return false;
    usleep(200);
  }
  return true;
}

// Waits until `flag` (&ShmSlot::hello or &ShmSlot::ready) is set in every rank's slot of the control block.
int wait_slots(const b2_comm* c, std::atomic<uint32_t> ShmSlot::*flag, double deadline) {
  for (int r = 0; r < c->d.world; ++r) {
    while ((c->shm->slot[r].*flag).load(std::memory_order_acquire) != 1) {
      if (now_s() > deadline) return fail(B2_ETIMEOUT, "rendezvous timed out waiting for rank %d on %s", r, c->shm_path.c_str());
      usleep(200);
    }
  }
  return B2_OK;
}

// What a kernel records in the status word: B2_ETIMEOUT (a peer wait gave up) or B2_EINVAL, which says (by status word 1,
// which k_p2p sets to kStatusP2p before it records B2_EINVAL):
constexpr const char* kA2aStatusText = "an all-to-all's split sizes disagreed across ranks or exceeded the per-pair limit";
constexpr const char* kP2pStatusText = "a point-to-point receive's byte count disagreed with its sender's";

const char* einval_text(const b2_comm* c) {
  return reinterpret_cast<volatile uint32_t*>(c->status_host)[1] == kStatusP2p ? kP2pStatusText : kA2aStatusText;
}

// A kernel that gave up waiting for a peer leaves the communicator's buffers and counters in an unknown state.  An
// all-to-all that gave up its exchange leaves them consistent, but the outputs of that call are not written.
int check_not_poisoned(const b2_comm* c) {
  const uint32_t s = *reinterpret_cast<volatile uint32_t*>(c->status_host);
  if (s == static_cast<uint32_t>(-B2_EINVAL)) return fail(B2_ESTATE, "communicator poisoned: %s", einval_text(c));
  if (s != 0) return fail(B2_ESTATE, "communicator poisoned by an earlier peer-wait timeout");
  return B2_OK;
}

// Multi-process multicast bring-up (after every rank has mapped every peer arena).  Any failure on any rank sets
// sb->mc_fail and every rank drops the NVLS path together; the P2P mappings are unaffected.
void setup_multicast(b2_comm* c, int sock, const std::string& sock_base, int stash_mc_fd, double deadline) {
  ShmBlock* sb = c->shm;
  const int W = c->d.world, rank = c->d.rank;
  const vmm::Driver& drv = vmm::driver();
  std::string why;
  int mc_fd = stash_mc_fd;
  bool ok = true;
  if (rank == 0) {
    const CUmulticastObjectProp mp = vmm::mc_prop(W, c->arena_bytes);
    CUresult r = drv.MulticastCreate(&c->mc.handle, &mp);
    if (r != CUDA_SUCCESS) {
      why = "cuMulticastCreate: " + vmm::errstr(r);
      ok = false;
    }
    int fd = -1;
    if (ok) {
      r = drv.MemExportToShareableHandle(&fd, c->mc.handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
      if (r != CUDA_SUCCESS) {
        why = "export of the multicast object: " + vmm::errstr(r);
        ok = false;
      }
    }
    for (int p = 1; p < W && ok; ++p) ok = vmm::send_fd(sock, sock_base, p, fd, vmm::FdMsg{0, 1}, &why);
    if (fd >= 0) close(fd);
  } else {
    while (mc_fd < 0 && ok) {
      if (sb->mc_fail.load(std::memory_order_acquire) || now_s() > deadline) {
        ok = false;
        why = "rank 0 could not create the multicast object";
        break;
      }
      vmm::FdMsg msg{};
      std::string w2;
      const int fd = vmm::recv_fd(sock, &msg, 100, &w2);
      if (fd >= 0 && msg.kind == 1) mc_fd = fd;
      else if (fd >= 0) close(fd);
    }
    if (ok) {
      const CUresult r = drv.MemImportFromShareableHandle(&c->mc.handle, reinterpret_cast<void*>(static_cast<uintptr_t>(mc_fd)),
                                                          CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
      if (r != CUDA_SUCCESS) {
        why = "import of the multicast object: " + vmm::errstr(r);
        ok = false;
      }
    }
    if (mc_fd >= 0) close(mc_fd);
  }
  CUdevice cudev = 0;
  if (ok && drv.DeviceGet(&cudev, c->device) != CUDA_SUCCESS) ok = false;
  if (ok) {
    const CUresult r = drv.MulticastAddDevice(c->mc.handle, cudev);
    if (r != CUDA_SUCCESS) {
      why = "cuMulticastAddDevice: " + vmm::errstr(r);
      ok = false;
    }
  }
  if (!ok) sb->mc_fail.store(1, std::memory_order_release);
  sb->mc_added.fetch_add(1, std::memory_order_acq_rel);
  ok = wait_count(sb->mc_added, W, nullptr, deadline) && !sb->mc_fail.load(std::memory_order_acquire) && ok;
  if (ok) {  // every device is in the team: binding cannot block
    const CUresult r = drv.MulticastBindMem(c->mc.handle, 0, c->own.handle, 0, c->arena_bytes, 0);
    if (r != CUDA_SUCCESS) {
      why = "cuMulticastBindMem: " + vmm::errstr(r);
      ok = false;
      sb->mc_fail.store(1, std::memory_order_release);
    }
  }
  sb->mc_bound.fetch_add(1, std::memory_order_acq_rel);
  ok = wait_count(sb->mc_bound, W, nullptr, deadline) && !sb->mc_fail.load(std::memory_order_acquire) && ok;
  if (ok) {
    const size_t gran = vmm::arena_granularity(c->device, W, true);
    const std::string e = vmm::map_handle(&c->mc, c->arena_bytes, gran, &c->device, 1);
    if (!e.empty()) {
      why = "mapping the multicast object: " + e;
      ok = false;
      sb->mc_fail.store(1, std::memory_order_release);
    }
  }
  sb->mc_mapped.fetch_add(1, std::memory_order_acq_rel);
  ok = wait_count(sb->mc_mapped, W, nullptr, deadline) && !sb->mc_fail.load(std::memory_order_acquire) && ok;
  if (ok) {
    c->d.mc = reinterpret_cast<uint8_t*>(c->mc.va);
  } else {
    vmm::unmap_release(&c->mc);
    c->d.mc = nullptr;
    if (!why.empty() && env_size("B2_VERBOSE", 0)) fprintf(stderr, "[b200ddp] rank %d: NVLS disabled: %s\n", rank, why.c_str());
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int b2_version(void) { return B2_ABI_VERSION; }

const char* b2_last_error(void) { return g_err.c_str(); }

int b2_comm_create_local(b2_comm_t** out, int world, const int* devices, size_t stage_bytes) {
  if (!out || !devices || world < 1 || world > B2_MAX_WORLD)
    return fail(B2_EINVAL, "b2_comm_create_local: bad arguments (world=%d)", world);
  int prev = -1;
  cudaGetDevice(&prev);
  b2_comm* cs[B2_MAX_WORLD] = {};
  int rc = B2_OK;
  // distinct devices -> VMM arenas visible to every device of the world (+ one multicast object); repeated devices
  // (all ranks on one GPU, the single-GPU parity topology) -> plain cudaMalloc, no multicast
  bool distinct = world > 1;
  for (int a = 0; a < world; ++a)
    for (int b = a + 1; b < world; ++b)
      if (devices[a] == devices[b]) distinct = false;
  bool use_vmm = distinct && env_size("B2_VMM", 1) != 0;
  bool use_mc = use_vmm && env_size("B2_NVLS", 1) != 0;
  for (int r = 0; r < world && use_vmm; ++r) {
    const vmm::Caps cp = vmm::caps(devices[r]);
    use_vmm = use_vmm && cp.vmm;
    use_mc = use_mc && cp.multicast;
  }
  use_mc = use_mc && use_vmm;
  for (int r = 0; r < world && rc == B2_OK; ++r) {
    cs[r] = new (std::nothrow) b2_comm();
    if (!cs[r]) {
      rc = fail(B2_ESYS, "out of host memory");
      break;
    }
    cs[r]->local_world = true;
    rc = init_rank(cs[r], r, world, devices[r], stage_bytes);
  }
  for (int a = 0; a < world && rc == B2_OK; ++a) {
    for (int b = 0; b < world && rc == B2_OK; ++b) {
      if (devices[a] == devices[b]) continue;
      int can = 0;
      cudaDeviceCanAccessPeer(&can, devices[a], devices[b]);
      if (!can) {
        rc = fail(B2_ENOPEER, "device %d cannot access device %d over P2P", devices[a], devices[b]);
        break;
      }
      cudaSetDevice(devices[a]);
      cudaError_t e = cudaDeviceEnablePeerAccess(devices[b], 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();
      } else if (e != cudaSuccess) {
        rc = fail(B2_ECUDA, "cudaDeviceEnablePeerAccess(%d->%d): %s", devices[a], devices[b],
                  cudaGetErrorString(e));
      }
    }
  }
  for (int r = 0; r < world && rc == B2_OK; ++r) rc = alloc_arena(cs[r], use_vmm, use_mc, devices, use_vmm ? world : 1);
  if (rc == B2_OK && use_mc) {
    // one multicast object over the W allocations, mapped once for all devices of the world
    const vmm::Driver& drv = vmm::driver();
    LocalMc* lm = new (std::nothrow) LocalMc();
    bool ok = lm != nullptr;
    if (ok) {
      const CUmulticastObjectProp mp = vmm::mc_prop(world, cs[0]->arena_bytes);
      ok = drv.MulticastCreate(&lm->map.handle, &mp) == CUDA_SUCCESS;
      for (int r = 0; r < world && ok; ++r) {
        CUdevice dv;
        ok = drv.DeviceGet(&dv, devices[r]) == CUDA_SUCCESS && drv.MulticastAddDevice(lm->map.handle, dv) == CUDA_SUCCESS;
      }
      for (int r = 0; r < world && ok; ++r)
        ok = drv.MulticastBindMem(lm->map.handle, 0, cs[r]->own.handle, 0, cs[r]->arena_bytes, 0) == CUDA_SUCCESS;
      if (ok) ok = vmm::map_handle(&lm->map, cs[0]->arena_bytes, vmm::arena_granularity(devices[0], world, true), devices, world).empty();
      if (ok) {
        lm->refs = world;
        for (int r = 0; r < world; ++r) {
          cs[r]->local_mc = lm;
          cs[r]->d.mc = reinterpret_cast<uint8_t*>(lm->map.va);
        }
      } else {
        vmm::unmap_release(&lm->map);
        delete lm;
      }
    }
  }
  if (rc == B2_OK) {
    for (int a = 0; a < world; ++a)
      for (int b = 0; b < world; ++b) cs[a]->arena_of[b] = static_cast<uint8_t*>(cs[b]->arena);
    for (int r = 0; r < world; ++r) {
      rotate_peers(cs[r]);
      out[r] = cs[r];
    }
  } else {
    std::string keep = g_err;
    for (int r = 0; r < world; ++r)
      if (cs[r]) {
        free_rank_resources(cs[r]);
        delete cs[r];
      }
    g_err = keep;
  }
  if (prev >= 0) cudaSetDevice(prev);
  return rc;
}

int b2_comm_create(b2_comm_t** out, int rank, int world, int device, const char* shm_name,
                   uint64_t epoch, size_t stage_bytes, int timeout_ms) {
  if (!out || world < 1 || world > B2_MAX_WORLD || rank < 0 || rank >= world || device < 0)
    return fail(B2_EINVAL, "b2_comm_create: bad arguments (rank=%d world=%d device=%d)", rank, world,
                device);
  if (world > 1 && (!shm_name || !*shm_name))
    return fail(B2_EINVAL, "b2_comm_create: shm_name is required when world > 1");
  const double deadline = now_s() + (timeout_ms > 0 ? timeout_ms : 120000) * 1e-3;
  int prev = -1;
  cudaGetDevice(&prev);
  b2_comm* c = new (std::nothrow) b2_comm();
  if (!c) return fail(B2_ESYS, "out of host memory");
  int rc = init_rank(c, rank, world, device, stage_bytes);
  int sock = -1;
  std::string sock_base;
  if (rc == B2_OK && world == 1) rc = alloc_arena(c, false, false, &device, 1);
  if (rc == B2_OK && world > 1) {
    // <name>.e<epoch>.c<n>: n counts this process's communicators on (name, epoch).  Every rank creates its
    // communicators in the same order, so n agrees across ranks, and a second communicator (init_pg + DDP, two DDP
    // modules) can never open the control block of the first one while rank 0 has not unlinked it yet.
    char path[256];
    snprintf(path, sizeof(path), "%s%s.e%llu.c%u", shm_name[0] == '/' ? "" : "/", shm_name,
             static_cast<unsigned long long>(epoch), next_creation_index(shm_name, epoch));
    c->shm_path = path;
    sock_base = std::string("b2fd") + path;
    int fd = shm_open(path, O_CREAT | O_RDWR, 0600);
    if (fd < 0) rc = fail(B2_ESYS, "shm_open(%s): %s", path, strerror(errno));
    if (rc == B2_OK && ftruncate(fd, sizeof(ShmBlock)) != 0)
      rc = fail(B2_ESYS, "ftruncate(%s): %s", path, strerror(errno));
    if (rc == B2_OK) {
      void* m = mmap(nullptr, sizeof(ShmBlock), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
      if (m == MAP_FAILED)
        rc = fail(B2_ESYS, "mmap(%s): %s", path, strerror(errno));
      else
        c->shm = static_cast<ShmBlock*>(m);
    }
    if (fd >= 0) close(fd);
  }
  if (rc == B2_OK && world > 1) {
    ShmBlock* sb = c->shm;
    ShmSlot& me = sb->slot[rank];
    // ---- 1. agree on the backend before anybody allocates -------------------------------------------------
    vmm::Caps cp;
    if (env_size("B2_VMM", 1) != 0) cp = vmm::caps(device);
    if (cp.vmm) {
      std::string why;
      sock = vmm::sock_open(sock_base, rank, &why);
      if (sock < 0) cp = vmm::Caps();  // no way to pass file descriptors: stay on CUDA IPC
    }
    if (env_size("B2_NVLS", 1) == 0) cp.multicast = false;
    me.cap_vmm = cp.vmm ? 1 : 0;
    me.cap_mc = cp.multicast ? 1 : 0;
    me.device = device;
    memset(me.bus_id, 0, sizeof(me.bus_id));
    cudaDeviceGetPCIBusId(me.bus_id, sizeof(me.bus_id), device);
    if (rank == 0) {
      sb->epoch = epoch;
      sb->world = world;
      sb->magic.store(kShmMagic, std::memory_order_release);
    }
    me.hello.store(1, std::memory_order_release);
    bool use_vmm = true, use_mc = true;
    rc = wait_slots(c, &ShmSlot::hello, deadline);
    for (int r = 0; r < world && rc == B2_OK; ++r) {
      use_vmm = use_vmm && sb->slot[r].cap_vmm != 0;
      use_mc = use_mc && sb->slot[r].cap_mc != 0;
    }
    // a multicast team is a set of DISTINCT devices: ranks sharing a GPU (functional tests) stay on the P2P kernels
    for (int a = 0; a < world && rc == B2_OK; ++a)
      for (int b = a + 1; b < world; ++b)
        if (strncmp(sb->slot[a].bus_id, sb->slot[b].bus_id, sizeof(sb->slot[a].bus_id)) == 0) use_mc = false;
    use_mc = use_mc && use_vmm;
    // ---- 2. allocate and publish ---------------------------------------------------------------------------
    if (rc == B2_OK) rc = alloc_arena(c, use_vmm, use_mc, &device, 1);
    if (rc == B2_OK) {
      if (!use_vmm) {
        cudaError_t e = cudaIpcGetMemHandle(&me.handle, c->arena);
        if (e != cudaSuccess) rc = fail(B2_ECUDA, "cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
      }
      me.pid = static_cast<int>(getpid());
      me.arena_bytes = c->arena_bytes;
      if (rc == B2_OK) me.ready.store(1, std::memory_order_release);
    }
    if (rc == B2_OK) rc = wait_slots(c, &ShmSlot::ready, deadline);
    // ---- 3. map every peer's arena -------------------------------------------------------------------------
    int stash_mc_fd = -1;
    for (int r = 0; r < world && rc == B2_OK; ++r) {
      if (r == rank) continue;
      const ShmSlot& ps = sb->slot[r];
      if (ps.arena_bytes != c->arena_bytes) {
        rc = fail(B2_EINVAL, "rank %d uses arena_bytes=%llu, this rank %zu (stage size must match)", r,
                  ps.arena_bytes, c->arena_bytes);
        break;
      }
      // Resolve the peer's GPU in THIS process's numbering by bus id.  If it is not visible here (each "node" of a
      // multi-node-on-one-box job gets its own CUDA_VISIBLE_DEVICES) the P2P query is impossible, but an IPC / imported
      // mapping of an invisible peer's memory can still be opened, so we just try.
      int peer_local = -1;
      if (cudaDeviceGetByPCIBusId(&peer_local, ps.bus_id) != cudaSuccess) {
        cudaGetLastError();
        peer_local = -1;
      }
      if (peer_local >= 0 && peer_local != device) {
        int can = 0;
        cudaDeviceCanAccessPeer(&can, device, peer_local);
        if (!can) {
          rc = fail(B2_ENOPEER, "device %d cannot access rank %d's device %s over P2P", device, r, ps.bus_id);
          break;
        }
      }
      if (!use_vmm) {
        void* p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, ps.handle, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
          rc = fail(B2_ECUDA, "cudaIpcOpenMemHandle(rank %d, device %d): %s", r, ps.device,
                    cudaGetErrorString(e));
          break;
        }
        c->arena_of[r] = static_cast<uint8_t*>(p);
        c->peer_is_ipc[r] = true;
      }
    }
    if (rc == B2_OK && use_vmm) {
      const vmm::Driver& drv = vmm::driver();
      std::string why;
      int fd = -1;
      CUresult r0 = drv.MemExportToShareableHandle(&fd, c->own.handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
      if (r0 != CUDA_SUCCESS) rc = fail(B2_ECUDA, "cuMemExportToShareableHandle: %s", vmm::errstr(r0).c_str());
      for (int p = 0; p < world && rc == B2_OK; ++p) {
        if (p == rank) continue;
        if (!vmm::send_fd(sock, sock_base, p, fd, vmm::FdMsg{rank, 0}, &why)) rc = fail(B2_ESYS, "%s", why.c_str());
      }
      if (fd >= 0) close(fd);
      int got = 0;
      const size_t gran = vmm::arena_granularity(device, world, use_mc);
      while (rc == B2_OK && got < world - 1) {
        if (now_s() > deadline) {
          rc = fail(B2_ETIMEOUT, "rendezvous timed out receiving peer arenas (%d/%d)", got, world - 1);
          break;
        }
        vmm::FdMsg msg{};
        const int pfd = vmm::recv_fd(sock, &msg, 200, &why);
        if (pfd < 0) continue;
        if (msg.kind == 1) {  // rank 0 is already at the multicast step
          stash_mc_fd = pfd;
          continue;
        }
        if (msg.src_rank < 0 || msg.src_rank >= world || msg.src_rank == rank || c->peers[msg.src_rank].handle) {
          close(pfd);
          continue;
        }
        vmm::Mapping& pm = c->peers[msg.src_rank];
        CUresult r1 = drv.MemImportFromShareableHandle(&pm.handle, reinterpret_cast<void*>(static_cast<uintptr_t>(pfd)),
                                                       CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
        close(pfd);
        if (r1 != CUDA_SUCCESS) {
          rc = fail(B2_ECUDA, "cuMemImportFromShareableHandle(rank %d): %s", msg.src_rank, vmm::errstr(r1).c_str());
          break;
        }
        const std::string e = vmm::map_handle(&pm, c->arena_bytes, gran, &device, 1);
        if (!e.empty()) {
          rc = fail(B2_ECUDA, "mapping rank %d's arena: %s", msg.src_rank, e.c_str());
          break;
        }
        c->arena_of[msg.src_rank] = reinterpret_cast<uint8_t*>(pm.va);
        ++got;
      }
    }
    if (rc == B2_OK) {
      sb->mapped.fetch_add(1, std::memory_order_acq_rel);
      if (!wait_count(sb->mapped, world, nullptr, deadline))
        rc = fail(B2_ETIMEOUT, "rendezvous timed out waiting for peers to map (%d/%d)", sb->mapped.load(), world);
    }
    // ---- 4. NVLS: one multicast object over all arenas -----------------------------------------------------
    if (rc == B2_OK && use_mc) setup_multicast(c, sock, sock_base, stash_mc_fd, deadline);
    else if (stash_mc_fd >= 0) close(stash_mc_fd);
    // everyone holds its mappings now: the name can go (the memory lives until the last munmap)
    if (rc == B2_OK && rank == 0) shm_unlink(c->shm_path.c_str());
  }
  if (sock >= 0) close(sock);
  if (rc != B2_OK) {
    std::string keep = g_err;
    for (int r = 0; r < world; ++r)
      if (c->peer_is_ipc[r]) cudaIpcCloseMemHandle(c->arena_of[r]);
    if (c->shm) munmap(c->shm, sizeof(ShmBlock));
    if (rank == 0 && !c->shm_path.empty()) shm_unlink(c->shm_path.c_str());
    free_rank_resources(c);
    delete c;
    g_err = keep;
  } else {
    rotate_peers(c);
    *out = c;
  }
  if (prev >= 0) cudaSetDevice(prev);
  return rc;
}

int b2_comm_destroy(b2_comm_t* c) {
  if (!c) return B2_OK;
  int prev = -1;
  cudaGetDevice(&prev);
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  if (c->shm) {
    // nobody frees its arena while a peer may still have kernels reading it
    ShmBlock* sb = c->shm;
    sb->departed.fetch_add(1, std::memory_order_acq_rel);
    const double deadline = now_s() + 10.0;
    while (sb->departed.load(std::memory_order_acquire) < c->d.world && now_s() < deadline) usleep(200);
    for (int r = 0; r < c->d.world; ++r)
      if (c->peer_is_ipc[r]) cudaIpcCloseMemHandle(c->arena_of[r]);
    munmap(c->shm, sizeof(ShmBlock));
  }
  free_rank_resources(c);
  delete c;
  if (prev >= 0) cudaSetDevice(prev);
  return B2_OK;
}

int b2_comm_rank(const b2_comm_t* c) { return c ? c->d.rank : B2_EINVAL; }
int b2_comm_world(const b2_comm_t* c) { return c ? c->d.world : B2_EINVAL; }
int b2_comm_device(const b2_comm_t* c) { return c ? c->device : B2_EINVAL; }

int b2_comm_caps(const b2_comm_t* c) {
  if (!c) return B2_EINVAL;
  return (c->use_vmm ? B2_CAP_VMM : 0) | (c->d.mc != nullptr ? B2_CAP_MULTICAST : 0);
}

int b2_comm_set_timeout_ms(b2_comm_t* c, int timeout_ms) {
  if (!c || timeout_ms <= 0) return fail(B2_EINVAL, "b2_comm_set_timeout_ms: bad arguments");
  c->d.timeout_ns = static_cast<unsigned long long>(timeout_ms) * 1000000ull;
  return B2_OK;
}

int b2_comm_set_max_ctas(b2_comm_t* c, int max_ctas) {
  if (!c || max_ctas < 0) return fail(B2_EINVAL, "b2_comm_set_max_ctas: bad arguments");
  c->max_ctas = max_ctas;
  return B2_OK;
}

int b2_comm_set_param(b2_comm_t* c, const char* name, long long value) {
  if (!c || !name || value < 0) return fail(B2_EINVAL, "b2_comm_set_param: bad arguments");
  const std::string k(name);
  if (k == "oneshot_max_bytes") c->policy.oneshot_max = static_cast<size_t>(value);
  else if (k == "pipe_min_bytes") c->policy.pipe_min = static_cast<size_t>(value);
  else if (k == "nvls_min_bytes") c->policy.nvls_min = static_cast<size_t>(value);
  else if (k == "nvls_min_world") c->policy.nvls_min_world = static_cast<int>(value);
  else if (k == "ll_min_bytes") c->policy.ll_min = static_cast<size_t>(value);
  else if (k == "ll_max_bytes") c->policy.ll_max = static_cast<size_t>(value);
  else if (k == "pipe_chunk_bytes") c->pipe_chunk_bytes = static_cast<size_t>(value);
  else if (k == "max_ctas") c->max_ctas = static_cast<int>(value);
  else if (k == "op_count") {
    const uint64_t v = static_cast<uint64_t>(value);
    DeviceGuard g(c->device);
    B2_CUDA(cudaDeviceSynchronize());  // the counter is only rewritten between collectives
    B2_CUDA(cudaMemcpy(c->d.opseq, &v, sizeof(v), cudaMemcpyHostToDevice));
  }
  else return fail(B2_EINVAL, "b2_comm_set_param: unknown parameter '%s'", name);
  return B2_OK;
}

uint64_t b2_comm_op_count(const b2_comm_t* c) {
  if (!c) {
    fail(B2_EINVAL, "b2_comm_op_count: null communicator");
    return 0;
  }
  uint64_t v = 0;
  DeviceGuard g(c->device);
  const cudaError_t e = cudaMemcpy(&v, c->d.opseq, sizeof(v), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) {
    fail(B2_ECUDA, "b2_comm_op_count: %s", cudaGetErrorString(e));
    return 0;
  }
  return v;
}

int b2_comm_status(const b2_comm_t* c) {
  if (!c) return fail(B2_EINVAL, "null communicator");
  const uint32_t s = *reinterpret_cast<volatile uint32_t*>(c->status_host);
  if (s == 0) return B2_OK;
  return fail(-static_cast<int>(s), "rank %d: %s (code %d)", c->d.rank,
              s == static_cast<uint32_t>(-B2_EINVAL) ? einval_text(c) : "a kernel gave up waiting for a peer", -static_cast<int>(s));
}

uint64_t b2_comm_launch_count(const b2_comm_t* c) { return c ? c->launches : 0; }

int b2_comm_last_algo(const b2_comm_t* c) { return c ? c->last_algo : B2_EINVAL; }

int b2_auto_algo(int world, int mode, size_t n_elems, int has_multicast) {
  if (world < 1 || world > B2_MAX_WORLD || !known_mode(mode))
    return fail(B2_EINVAL, "b2_auto_algo: bad arguments (world=%d mode=%d)", world, mode);
  if (world == 1 || n_elems == 0) return B2_ALGO_AUTO;  // no collective: the local pass
  const size_t wire = (n_elems + 7) / 8 * wire_vec_bytes(mode);
  return auto_algo(default_policy(world), world, mode, wire, has_multicast != 0, true);
}

int b2_comm_trace(b2_comm_t* c, int enable, uint64_t* out, int max_ctas) {
  if (!c) return fail(B2_EINVAL, "null communicator");
  DeviceGuard g(c->device);
  if (enable && !c->trace_dev) B2_CUDA(cudaMalloc(&c->trace_dev, sizeof(unsigned long long) * kMaxCtas * 8));
  if (out && max_ctas > 0 && c->trace_dev) {
    const int n = max_ctas < kMaxCtas ? max_ctas : kMaxCtas;
    B2_CUDA(cudaMemcpy(out, c->trace_dev, sizeof(unsigned long long) * n * 8, cudaMemcpyDeviceToHost));
  }
  if (enable) B2_CUDA(cudaMemset(c->trace_dev, 0, sizeof(unsigned long long) * kMaxCtas * 8));  // no stale CTAs
  c->d.trace = enable ? c->trace_dev : nullptr;
  return B2_OK;
}

int b2_local_pass(void* buf, size_t n_elems, int mode, float scale, int device, void* stream) {
  return local_pass_impl(kNoSrc, buf, n_elems, mode, scale, device, stream);
}

static int allreduce_impl(b2_comm_t* c, Src& src, void* buf, size_t n_elems, int mode, float scale, int algo, void* stream) {
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!known_mode(mode)) return fail(B2_EINVAL, "unknown mode %d", mode);
  if (algo != B2_ALGO_AUTO && algo != B2_ALGO_ONESHOT && algo != B2_ALGO_TWOSHOT && algo != B2_ALGO_TWOSHOT_PIPE &&
      algo != B2_ALGO_NVLS && algo != B2_ALGO_TWOSHOT_LL)
    return fail(B2_EINVAL, "unknown algo %d", algo);
  if (n_elems == 0) return B2_OK;
  if (!buf) return fail(B2_EINVAL, "b2_allreduce: null buffer");
  if (const int rc = check_not_poisoned(c)) return rc;
  const int W = c->d.world;
  if (W == 1) {
    if (mode == B2_F32 && scale == 1.0f && src.nseg == 0) return B2_OK;  // identity
    int rc = local_pass_impl(src, buf, n_elems, mode, scale, c->device, stream);
    if (rc == B2_OK) c->launches++;
    return rc;
  }
  if (algo == B2_ALGO_NVLS && c->d.mc == nullptr)
    return fail(B2_ENOTSUP, "B2_ALGO_NVLS: this communicator has no multicast mapping (b2_comm_caps)");
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t wvb = wire_vec_bytes(mode);
  const size_t cap_vecs = c->d.slice_cap / wvb;  // vecs one region can hold
  const int U = vecs_per_trip(W);
  uint8_t* p = static_cast<uint8_t*>(buf);
  size_t left = n_elems;
  while (left > 0) {
    const unsigned long long V_left = (left + 7) / 8;
    const size_t wire_left = V_left * wvb;
    int kind;
    if (algo == B2_ALGO_AUTO) {
      kind = auto_algo(c->policy, W, mode, wire_left, c->d.mc != nullptr, V_left <= cap_vecs);
    } else {
      kind = algo;
    }
    const bool oneshot = kind == B2_ALGO_ONESHOT;
    const unsigned long long max_vecs = oneshot ? cap_vecs : cap_vecs * W;
    const unsigned long long V = V_left < max_vecs ? V_left : max_vecs;
    const size_t n = V == V_left ? left : static_cast<size_t>(V) * 8;
    const unsigned long long Ls = (V + W - 1) / W;
    const PipePlan plan = plan_pipe(c, Ls, V * wvb);
    const int grid = grid_for(c, oneshot ? V : Ls, U);
    cudaError_t e = cudaErrorInvalidValue;  // never guess a mode
    with_mode(mode, [&](auto m) { e = launch_collective<decltype(m)::value>(c->d, src, kind, grid, plan, p, n, scale, s); });
    if (e != cudaSuccess) return fail(B2_ECUDA, "allreduce kernel launch: %s", cudaGetErrorString(e));
    c->launches++;
    c->last_algo = kind;
    p += n * elem_bytes(mode);
    src.off += n;
    left -= n;
  }
  return B2_OK;
}

int b2_allreduce(b2_comm_t* c, void* buf, size_t n_elems, int mode, float scale, int algo, void* stream) {
  Src src = kNoSrc;
  return allreduce_impl(c, src, buf, n_elems, mode, scale, algo, stream);
}

// The segment table of a gather call -> `src`: 1..B2_MAX_SEGMENTS entries that cover bucket elements [0, n_elems) in
// order and without gaps, each with a source pointer or B2_SEGMENT_ZEROS, which the device table holds as a null pointer
// (load_src reads such a segment as +0.0).  `fn` names the call in the error texts.
static int segment_table(const char* fn, const b2_segment_t* segments, int n_segments, size_t n_elems, Src& src) {
  if (!segments || n_segments <= 0 || n_segments > B2_MAX_SEGMENTS)
    return fail(B2_EINVAL, "%s: need 1..%d segments (got %d)", fn, B2_MAX_SEGMENTS, n_segments);
  src.nseg = n_segments;
  src.off = 0;
  unsigned long long at = 0;
  for (int i = 0; i < n_segments; ++i) {
    if (segments[i].begin != at || segments[i].end <= at || !segments[i].src)
      return fail(B2_EINVAL, "%s: segment %d does not continue the bucket at element %llu", fn, i, at);
    src.ptr[i] = segments[i].src == B2_SEGMENT_ZEROS ? nullptr : segments[i].src;
    src.begin[i] = at;
    at = segments[i].end;
  }
  if (at != n_elems) return fail(B2_EINVAL, "%s: segments cover %llu elements, bucket has %zu", fn, at, n_elems);
  for (int i = n_segments; i <= B2_MAX_SEGMENTS; ++i) src.begin[i] = at;
  for (int i = n_segments; i < B2_MAX_SEGMENTS; ++i) src.ptr[i] = nullptr;
  return B2_OK;
}

int b2_allreduce_gather(b2_comm_t* c, void* out, size_t n_elems, const b2_segment_t* segments, int n_segments, int mode,
                        float scale, int algo, void* stream) {
  if (n_elems == 0) return B2_OK;
  Src src;
  if (const int rc = segment_table("b2_allreduce_gather", segments, n_segments, n_elems, src)) return rc;
  return allreduce_impl(c, src, out, n_elems, mode, scale, algo, stream);
}

int b2_reduce_scatter_gather(b2_comm_t* c, void* out, size_t block, const b2_segment_t* segments, int n_segments, int mode,
                             float scale, void* stream) {
  if (!known_mode(mode)) return fail(B2_EINVAL, "b2_reduce_scatter_gather: unknown mode %d", mode);
  if (block == 0) return B2_OK;
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!out) return fail(B2_EINVAL, "b2_reduce_scatter_gather: null buffer");
  const int W = c->d.world;
  Src src;
  if (const int rc = segment_table("b2_reduce_scatter_gather", segments, n_segments, static_cast<size_t>(W) * block, src)) return rc;
  if (const int rc = check_not_poisoned(c)) return rc;
  if (W == 1) {  // the local pass of b2_allreduce_gather, rounding included
    const int rc = local_pass_impl(src, out, block, mode, scale, c->device, stream);
    if (rc == B2_OK) c->launches++;
    return rc;
  }
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t eb = elem_bytes(mode);
  const size_t cap = c->d.slice_cap / wire_vec_bytes(mode) * 8;  // elements of a block one recv region holds (whole vecs)
  uint8_t* po = static_cast<uint8_t*>(out);
  const cudaError_t e = for_chunks(c, block, cap, [&](size_t off, size_t n) {
    const int grid = grid_for(c, (n + 7) / 8, vecs_per_trip(W));
    src.off = off;  // every block's launch-local element 0 is bucket element j * block + off
    cudaError_t le = cudaErrorInvalidValue;  // never guess a mode
    with_mode(mode, [&](auto m) {
      le = launch_reduce_scatter<decltype(m)::value>(c->d, src, grid, po + off * eb, nullptr, n, block, scale, s);
    });
    return le;
  });
  if (e != cudaSuccess) return fail(B2_ECUDA, "reduce-scatter kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

// b2_optim_t -> the kernels' OptDev: the hyper-parameters rounded to fp32 as ATen's fused launches round them, the runs
// checked to tile [0, block).  `fn` names the call in the error texts.
static int optim_table(const char* fn, const b2_optim_t* opt, size_t block, OptDev& o) {
  if (!opt) return fail(B2_EINVAL, "%s: null optimizer", fn);
  if (opt->kind != B2_OPT_SGD && opt->kind != B2_OPT_ADAM && opt->kind != B2_OPT_ADAMW)
    return fail(B2_EINVAL, "%s: unknown optimizer kind %d", fn, opt->kind);
  if (opt->n_groups <= 0 || opt->n_groups > B2_OPT_MAX_GROUPS)
    return fail(B2_EINVAL, "%s: need 1..%d parameter groups (got %d)", fn, B2_OPT_MAX_GROUPS, opt->n_groups);
  if (opt->n_runs <= 0 || opt->n_runs > B2_OPT_MAX_RUNS)
    return fail(B2_EINVAL, "%s: need 1..%d runs (got %d)", fn, B2_OPT_MAX_RUNS, opt->n_runs);
  if (block >= (1ull << 32)) return fail(B2_EINVAL, "%s: block of %zu elements (the runs are 32-bit)", fn, block);
  const bool adam = opt->kind != B2_OPT_SGD;
  bool momentum = false;
  o.kind = opt->kind;
  o.nrun = opt->n_runs;
  for (int gi = 0; gi < B2_OPT_MAX_GROUPS; ++gi) {
    OptGroupDev& g = o.g[gi];
    g = OptGroupDev{};
    if (gi >= opt->n_groups) continue;
    const b2_optim_group_t& h = opt->group[gi];
    g.lr = static_cast<float>(h.lr);
    g.wd = static_cast<float>(h.weight_decay);
    g.flags = (h.maximize ? B2_OPT_F_MAXIMIZE : 0);
    if (adam) {
      g.a = static_cast<float>(h.beta1);
      g.b = static_cast<float>(h.beta2);
      g.eps = static_cast<float>(h.eps);
      g.lr_wd = g.lr * g.wd;  // fp32 product, as ATen's AdamW forms it
    } else {
      g.a = static_cast<float>(h.momentum);
      g.b = 1.0f - static_cast<float>(h.dampening);  // fp32, as the fused SGD kernel forms it
      g.flags |= (h.nesterov ? B2_OPT_F_NESTEROV : 0) | (h.momentum != 0.0 ? B2_OPT_F_MOMENTUM : 0);
      momentum = momentum || h.momentum != 0.0;
    }
  }
  if (!opt->param || ((adam || momentum) && !opt->state0) || (adam && !opt->state1))
    return fail(B2_EINVAL, "%s: null parameter or state pointer", fn);
  o.param = opt->param;
  o.s0 = opt->state0 ? opt->state0 : opt->param;  // never dereferenced without momentum
  o.s1 = opt->state1 ? opt->state1 : opt->param;
  o.off = 0;
  if (opt->run_begin[0] != 0 || opt->run_begin[opt->n_runs] != block)
    return fail(B2_EINVAL, "%s: runs cover [%llu, %llu), the block is [0, %zu)", fn, (unsigned long long)opt->run_begin[0],
                (unsigned long long)opt->run_begin[opt->n_runs], block);
  for (int k = 0; k < opt->n_runs; ++k) {
    if (opt->run_begin[k + 1] <= opt->run_begin[k]) return fail(B2_EINVAL, "%s: run %d is empty or out of order", fn, k);
    const int gi = opt->run_group[k];
    if (gi != B2_OPT_NO_GROUP && gi >= opt->n_groups) return fail(B2_EINVAL, "%s: run %d names group %d of %d", fn, k, gi, opt->n_groups);
    o.begin[k] = static_cast<uint32_t>(opt->run_begin[k]);
    o.group[k] = static_cast<uint8_t>(gi | (gi != B2_OPT_NO_GROUP && opt->run_scalar[k] ? kOptScalar : 0));
    o.pidx[k] = static_cast<uint16_t>(opt->run_index[k] & 0xffffu);
    o.step[k] = opt->run_step[k];
  }
  for (int k = opt->n_runs; k <= B2_OPT_MAX_RUNS; ++k) o.begin[k] = static_cast<uint32_t>(block);
  for (int k = opt->n_runs; k < B2_OPT_MAX_RUNS; ++k) {
    o.group[k] = B2_OPT_NO_GROUP;
    o.pidx[k] = 0;
    o.step[k] = 0.f;
  }
  return B2_OK;
}

// The launches of one fused step, fp32 bucket or bf16 bucket: at W == 1 the local pass's grid and rounding, else one
// reduce-scatter step kernel per stage-sized piece of the block.
extern "C++" template <int MODE>
cudaError_t launch_step(b2_comm* c, Src& src, typename OptOf<MODE>::type& o, size_t block, float scale, void* stream) {
  const int W = c->d.world;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (W == 1) {
    k_local_step<MODE><<<local_grid(block, sm_count(c->device)), kThreads, 0, s>>>(src, o, block, scale);
    c->launches++;
    return cudaGetLastError();
  }
  const size_t cap = c->d.slice_cap / dev::Wire<MODE>::kBytes * 8;  // elements of a block one recv region holds
  return for_chunks(c, block, cap, [&](size_t off, size_t n) {
    src.off = off;  // the same block offset for the gradient table and the parameter / state slices
    o.off = off;
    cudaError_t le = cudaErrorInvalidValue;
    with_world(W, [&](auto w) {
      k_reduce_scatter_step<MODE, decltype(w)::value><<<grid_for(c, (n + 7) / 8, 1), kThreads, 0, s>>>(c->d, src, o, n, block, scale);
      le = cudaGetLastError();
    });
    return le;
  });
}

int b2_reduce_scatter_step(b2_comm_t* c, size_t block, const b2_segment_t* segments, int n_segments, int mode, float scale,
                           const b2_optim_t* opt, void* stream) {
  if (mode != B2_F32_WIRE_BF16 && mode != B2_F32 && mode != B2_F32_WIRE_F16)
    return fail(B2_EINVAL, "b2_reduce_scatter_step: mode %d (fp32 buckets only: modes 0, 1, 3)", mode);
  if (block == 0) return B2_OK;
  OptDev o;  // checked first: it needs no communicator
  if (const int rc = optim_table("b2_reduce_scatter_step", opt, block, o)) return rc;
  if (!c) return fail(B2_EINVAL, "null communicator");
  const int W = c->d.world;
  Src src;
  if (const int rc = segment_table("b2_reduce_scatter_step", segments, n_segments, static_cast<size_t>(W) * block, src)) return rc;
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  cudaError_t e = cudaErrorInvalidValue;
  with_mode(mode, [&](auto m) {
    constexpr int MODE = decltype(m)::value;
    if constexpr (!k16BitBucket<MODE>) e = launch_step<MODE>(c, src, o, block, scale, stream);
  });
  if (e != cudaSuccess) return fail(B2_ECUDA, "reduce-scatter step kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_reduce_scatter_step_bf16(b2_comm_t* c, size_t block, const b2_segment_t* segments, int n_segments, float scale,
                                const b2_optim_t* opt, void* param_bf16, void* stream) {
  if (block == 0) return B2_OK;
  OptDevBf16 o;  // checked first: it needs no communicator
  if (const int rc = optim_table("b2_reduce_scatter_step_bf16", opt, block, o)) return rc;
  if (!param_bf16) return fail(B2_EINVAL, "b2_reduce_scatter_step_bf16: null bf16 parameter pointer");
  if (reinterpret_cast<uintptr_t>(param_bf16) & 15u)
    return fail(B2_EINVAL, "b2_reduce_scatter_step_bf16: bf16 parameter pointer not 16-byte aligned");
  o.pbf = static_cast<uint16_t*>(param_bf16);
  if (!c) return fail(B2_EINVAL, "null communicator");
  const int W = c->d.world;
  Src src;
  if (const int rc = segment_table("b2_reduce_scatter_step_bf16", segments, n_segments, static_cast<size_t>(W) * block, src)) return rc;
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  const cudaError_t e = launch_step<B2_BF16>(c, src, o, block, scale, stream);
  if (e != cudaSuccess) return fail(B2_ECUDA, "reduce-scatter step kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_broadcast(b2_comm_t* c, void* buf, size_t bytes, int root, void* stream) {
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (root < 0 || root >= c->d.world) return fail(B2_EINVAL, "b2_broadcast: root %d out of range", root);
  if (bytes == 0 || c->d.world == 1) return B2_OK;
  if (!buf) return fail(B2_EINVAL, "b2_broadcast: null buffer");
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t cap = c->stage_bytes & ~static_cast<size_t>(15);
  const cudaError_t e = for_chunks(c, bytes, cap, [&](size_t off, size_t n) {
    k_broadcast<<<grid_for(c, (n + 15) / 16, 1), kThreads, 0, s>>>(c->d, static_cast<uint8_t*>(buf) + off, n, root);
    return cudaGetLastError();
  });
  if (e != cudaSuccess) return fail(B2_ECUDA, "broadcast kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

}  // extern "C"

namespace {

// The B2_DT_* dtypes of include/b200ddp.h: calls f(std::integral_constant<int, DT>{}) and returns true, or returns false
// for an unknown dtype.  The only switch over them; what they are is exact::DtypeTraits<DT>.
template <class F>
bool with_dtype(int dtype, F&& f) {
  switch (dtype) {
    case B2_DT_INT32: f(std::integral_constant<int, B2_DT_INT32>{}); return true;
    case B2_DT_INT64: f(std::integral_constant<int, B2_DT_INT64>{}); return true;
    case B2_DT_FLOAT32: f(std::integral_constant<int, B2_DT_FLOAT32>{}); return true;
    case B2_DT_BFLOAT16: f(std::integral_constant<int, B2_DT_BFLOAT16>{}); return true;
    case B2_DT_FLOAT16: f(std::integral_constant<int, B2_DT_FLOAT16>{}); return true;
    default: return false;
  }
}

const char* dtype_name(int dtype) {
  const char* s = nullptr;
  with_dtype(dtype, [&](auto d) { s = exact::DtypeTraits<decltype(d)::value>::kName; });
  return s;
}

size_t dtype_bytes(int dtype) {
  size_t b = 0;
  with_dtype(dtype, [&](auto d) { b = exact::DtypeTraits<decltype(d)::value>::kBytes; });
  return b;
}

bool dtype_is_int(int dtype) {
  bool i = false;
  with_dtype(dtype, [&](auto d) { i = exact::DtypeTraits<decltype(d)::value>::kInt; });
  return i;
}

// The (dtype, op) pairs of the exact kernels: calls f(std::integral_constant<int, DT>{}, std::integral_constant<int, OP>{})
// and returns true, or returns false for float SUM / AVG and anything unknown.
template <class F>
bool with_exact_op(int dtype, int op, F&& f) {
  bool ok = false;
  with_dtype(dtype, [&](auto d) {
    switch (op) {
      case B2_OP_SUM:
        if constexpr (exact::DtypeTraits<decltype(d)::value>::kInt) {  // float SUM runs on the allreduce kernels
          f(d, std::integral_constant<int, B2_OP_SUM>{});
          ok = true;
        }
        break;
      case B2_OP_MIN:
        f(d, std::integral_constant<int, B2_OP_MIN>{});
        ok = true;
        break;
      case B2_OP_MAX:
        f(d, std::integral_constant<int, B2_OP_MAX>{});
        ok = true;
        break;
    }
  });
  return ok;
}

cudaError_t launch_reduce_exact(int dtype, int op, const CommDev& d, int grid, void* buf, unsigned long long n, cudaStream_t s) {
  cudaError_t e = cudaErrorInvalidValue;
  with_exact_op(dtype, op, [&](auto dt, auto o) {
    k_reduce_exact<decltype(dt)::value, decltype(o)::value><<<grid, kThreads, 0, s>>>(d, buf, n);
    e = cudaGetLastError();
  });
  return e;
}

// The B2_* mode of a float SUM / AVG: the gradient mode whose bucket has this dtype and is its own wire format.
int sum_mode_for(int dtype) { return dtype == B2_DT_FLOAT32 ? B2_F32 : (dtype == B2_DT_BFLOAT16 ? B2_BF16 : B2_F16); }

// Shared argument checks of b2_allreduce_op and b2_reduce_scatter, in their order: dtype, op, AVG on an integer dtype.
int check_dtype_op(const char* fn, int dtype, int op) {
  const char* dt = dtype_name(dtype);
  if (!dt) return fail(B2_EINVAL, "%s: unknown dtype %d", fn, dtype);
  if (op != B2_OP_SUM && op != B2_OP_AVG && op != B2_OP_MIN && op != B2_OP_MAX) return fail(B2_EINVAL, "%s: unknown op %d", fn, op);
  if (dtype_is_int(dtype) && op == B2_OP_AVG) return fail(B2_EINVAL, "%s: AVG needs a floating-point dtype, got %s", fn, dt);
  return B2_OK;
}

}  // namespace

extern "C" {

int b2_allreduce_op(b2_comm_t* c, void* buf, size_t n_elems, int dtype, int op, void* stream) {
  if (const int rc = check_dtype_op("b2_allreduce_op", dtype, op)) return rc;
  if (n_elems == 0) return B2_OK;
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!buf) return fail(B2_EINVAL, "b2_allreduce_op: null buffer");
  if (const int rc = check_not_poisoned(c)) return rc;
  const int W = c->d.world;
  if (W == 1) return B2_OK;
  if (!dtype_is_int(dtype) && (op == B2_OP_SUM || op == B2_OP_AVG)) {  // the rank-order fp32 sum of the gradient allreduce
    const int mode = sum_mode_for(dtype);
    Src src = kNoSrc;
    return allreduce_impl(c, src, buf, n_elems, mode, op == B2_OP_AVG ? 1.0f / static_cast<float>(W) : 1.0f, B2_ALGO_AUTO, stream);
  }
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t eb = dtype_bytes(dtype);
  const size_t cap = c->d.slice_cap / eb;  // elements one recv region holds (slice_cap is a multiple of 256 bytes)
  const cudaError_t e = for_chunks(c, n_elems, cap, [&](size_t off, size_t n) {
    return launch_reduce_exact(dtype, op, c->d, grid_for(c, (n * eb + 15) / 16, 1), static_cast<uint8_t*>(buf) + off * eb, n, s);
  });
  if (e != cudaSuccess) return fail(B2_ECUDA, "exact allreduce kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_allgather(b2_comm_t* c, void* out, const void* in, size_t bytes, void* stream) {
  if (bytes == 0) return B2_OK;
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!out || !in) return fail(B2_EINVAL, "b2_allgather: null buffer");
  const int W = c->d.world;
  const bool in_place = in == static_cast<const uint8_t*>(out) + static_cast<size_t>(c->d.rank) * bytes;
  if (!in_place && overlaps(in, bytes, out, static_cast<size_t>(W) * bytes))
    return fail(B2_EINVAL, "b2_allgather: `in` overlaps `out` other than as this rank's block");
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (W == 1) {
    if (!in_place) B2_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, s));
    return B2_OK;
  }
  const cudaError_t e = for_chunks(c, bytes, c->d.slice_cap, [&](size_t off, size_t n) {
    k_allgather<<<grid_for(c, (n + 15) / 16, 1), kThreads, 0, s>>>(c->d, static_cast<uint8_t*>(out) + off,
                                                                   static_cast<const uint8_t*>(in) + off, n, bytes);
    return cudaGetLastError();
  });
  if (e != cudaSuccess) return fail(B2_ECUDA, "all-gather kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_reduce_scatter(b2_comm_t* c, void* out, const void* in, size_t n_elems, int dtype, int op, void* stream) {
  if (const int rc = check_dtype_op("b2_reduce_scatter", dtype, op)) return rc;
  if (n_elems == 0) return B2_OK;
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!out || !in) return fail(B2_EINVAL, "b2_reduce_scatter: null buffer");
  const int W = c->d.world;
  const size_t eb = dtype_bytes(dtype);
  const size_t bytes = n_elems * eb;  // one block
  const bool in_place = out == static_cast<const uint8_t*>(in) + static_cast<size_t>(c->d.rank) * bytes;
  if (!in_place && overlaps(out, bytes, in, static_cast<size_t>(W) * bytes))
    return fail(B2_EINVAL, "b2_reduce_scatter: `out` overlaps `in` other than as this rank's block");
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (W == 1) {
    if (!in_place) B2_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, s));
    return B2_OK;
  }
  const bool sum = !dtype_is_int(dtype) && (op == B2_OP_SUM || op == B2_OP_AVG);
  const int mode = sum_mode_for(dtype);
  // elements of a block one recv region holds: a whole number of vecs in either case (slice_cap is a multiple of 256 bytes)
  const size_t cap = sum ? c->d.slice_cap / wire_vec_bytes(mode) * 8 : c->d.slice_cap / eb;
  const float scale = op == B2_OP_AVG ? 1.0f / static_cast<float>(W) : 1.0f;
  uint8_t* po = static_cast<uint8_t*>(out);
  const uint8_t* pi = static_cast<const uint8_t*>(in);
  const cudaError_t e = for_chunks(c, n_elems, cap, [&](size_t off, size_t n) {
    cudaError_t le = cudaErrorInvalidValue;  // never guess a mode
    if (sum) {
      const int grid = grid_for(c, (n + 7) / 8, vecs_per_trip(W));
      with_mode(mode, [&](auto m) {
        le = launch_reduce_scatter<decltype(m)::value>(c->d, kNoSrc, grid, po + off * eb, pi + off * eb, n, n_elems, scale, s);
      });
    } else {
      const int grid = grid_for(c, (n * eb + 15) / 16, 1);
      with_exact_op(dtype, op, [&](auto dt, auto oc) {
        k_reduce_scatter_exact<decltype(dt)::value, decltype(oc)::value><<<grid, kThreads, 0, s>>>(c->d, po + off * eb, pi + off * eb,
                                                                                                 n, n_elems);
        le = cudaGetLastError();
      });
    }
    return le;
  });
  if (e != cudaSuccess) return fail(B2_ECUDA, "reduce-scatter kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_reduce(b2_comm_t* c, void* buf, size_t n_elems, int dtype, int op, int root, void* stream) {
  if (const int rc = check_dtype_op("b2_reduce", dtype, op)) return rc;
  if (n_elems == 0) return B2_OK;
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!buf) return fail(B2_EINVAL, "b2_reduce: null buffer");
  const int W = c->d.world;
  if (root < 0 || root >= W) return fail(B2_EINVAL, "b2_reduce: root %d is not a rank of a world of %d", root, W);
  if (const int rc = check_not_poisoned(c)) return rc;
  if (W == 1) return B2_OK;
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool sum = !dtype_is_int(dtype) && (op == B2_OP_SUM || op == B2_OP_AVG);
  const int mode = sum_mode_for(dtype);
  const size_t eb = dtype_bytes(dtype);
  // the two-shot allreduce's plan: a launch holds W slices of at most one recv region each (whole vecs in either case)
  const size_t cap = sum ? c->d.slice_cap / wire_vec_bytes(mode) * 8 * W : c->d.slice_cap / 16 * W * (16 / eb);
  const float scale = op == B2_OP_AVG ? 1.0f / static_cast<float>(W) : 1.0f;
  uint8_t* p = static_cast<uint8_t*>(buf);
  const cudaError_t e = for_chunks(c, n_elems, cap, [&](size_t off, size_t n) {
    cudaError_t le = cudaErrorInvalidValue;  // never guess a mode
    if (sum) {
      const unsigned long long Ls = ((n + 7) / 8 + W - 1) / W;
      with_mode(mode, [&](auto m) {
        constexpr int MODE = decltype(m)::value;
        if constexpr (MODE == B2_F32 || MODE == B2_BF16 || MODE == B2_F16) {  // the modes sum_mode_for picks
          with_world(W, [&](auto w) {
            k_reduce<MODE, decltype(w)::value><<<grid_for(c, Ls, vecs_per_trip(W)), kThreads, 0, s>>>(c->d, p + off * eb, n, scale, root);
            le = cudaGetLastError();
          });
        }
      });
    } else {
      const unsigned long long Ls = ((n * eb + 15) / 16 + W - 1) / W;
      with_exact_op(dtype, op, [&](auto dt, auto oc) {
        k_reduce_exact_root<decltype(dt)::value, decltype(oc)::value><<<grid_for(c, Ls, 1), kThreads, 0, s>>>(c->d, p + off * eb, n, root);
        le = cudaGetLastError();
      });
    }
    return le;
  });
  if (e != cudaSuccess) return fail(B2_ECUDA, "reduce kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

size_t b2_alltoall_max_bytes(const b2_comm_t* c) { return c ? c->d.slice_cap - kA2aHeaderBytes : 0; }

int b2_alltoall(b2_comm_t* c, void* const* out, const size_t* recv_bytes, const void* const* in, const size_t* send_bytes,
                void* stream) {
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!out || !recv_bytes || !in || !send_bytes) return fail(B2_EINVAL, "b2_alltoall: null array");
  const int W = c->d.world, me = c->d.rank;
  for (int r = 0; r < W; ++r) {
    if (!out[r] && recv_bytes[r]) return fail(B2_EINVAL, "b2_alltoall: out[%d] is null but recv_bytes[%d] = %zu", r, r, recv_bytes[r]);
    if (!in[r] && send_bytes[r]) return fail(B2_EINVAL, "b2_alltoall: in[%d] is null but send_bytes[%d] = %zu", r, r, send_bytes[r]);
  }
  for (int r = 0; r < W; ++r) {
    for (int s = r + 1; s < W; ++s)
      if (overlaps(out[r], recv_bytes[r], out[s], recv_bytes[s])) return fail(B2_EINVAL, "b2_alltoall: out[%d] overlaps out[%d]", r, s);
    for (int j = 0; j < W; ++j)
      if (overlaps(out[r], recv_bytes[r], in[j], send_bytes[j])) return fail(B2_EINVAL, "b2_alltoall: out[%d] overlaps in[%d]", r, j);
  }
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (W == 1) {
    if (send_bytes[0] != recv_bytes[0])
      return fail(B2_EINVAL, "b2_alltoall: rank 0 sends %zu bytes to itself but expects %zu", send_bytes[0], recv_bytes[0]);
    if (recv_bytes[0]) B2_CUDA(cudaMemcpyAsync(out[0], in[0], recv_bytes[0], cudaMemcpyDeviceToDevice, s));
    return B2_OK;
  }
  // A pair over the limit is seen here by its sender and its receiver.  Both still launch, with the abort flag, so that no
  // rank waits for them and every rank's kernel sees the abort after its barrier.
  const size_t max = b2_alltoall_max_bytes(c);
  A2aArgs a{};
  int rc = B2_OK;
  for (int jj = 0; jj < W; ++jj) {
    const int r = (me + jj) % W;
    a.send[jj] = static_cast<const uint8_t*>(in[r]);
    a.send_bytes[jj] = send_bytes[r];
    a.recv[jj] = static_cast<uint8_t*>(out[r]);
    a.recv_bytes[jj] = recv_bytes[r];
    if (jj > 0 && rc == B2_OK && (send_bytes[r] > max || recv_bytes[r] > max))
      rc = fail(B2_EINVAL, "b2_alltoall: rank %d sends %zu bytes to rank %d and expects %zu from it; one pair carries at most %zu "
                "(a larger stage raises the limit: B2_STAGE_MB / stage_mb)", me, send_bytes[r], r, recv_bytes[r], max);
  }
  a.abort = rc != B2_OK;
  k_alltoall<<<grid_for(c, (max + 15) / 16, 1), kThreads, 0, s>>>(c->d, a);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "all-to-all kernel launch: %s", cudaGetErrorString(e));
  c->launches++;
  return rc;
}

size_t b2_p2p_eager_bytes(const b2_comm_t* c) { return c ? kP2pSlots * kP2pPayload : 0; }

int b2_p2p(b2_comm_t* c, const b2_p2p_op_t* ops, int n_ops, void* stream) {
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (!ops) return fail(B2_EINVAL, "b2_p2p: null op list");
  if (n_ops < 1 || n_ops > B2_P2P_MAX_OPS) return fail(B2_EINVAL, "b2_p2p: need 1..%d ops (got %d)", B2_P2P_MAX_OPS, n_ops);
  const int W = c->d.world, me = c->d.rank;
  for (int i = 0; i < n_ops; ++i) {
    if (ops[i].peer < 0 || ops[i].peer >= W || ops[i].peer == me)
      return fail(B2_EINVAL, "b2_p2p: op %d names peer %d; rank %d of %d can only name another rank", i, ops[i].peer, me, W);
    if (!ops[i].ptr && ops[i].bytes) return fail(B2_EINVAL, "b2_p2p: op %d has a null pointer and %zu bytes", i, ops[i].bytes);
  }
  for (int i = 0; i < n_ops; ++i) {
    if (ops[i].is_send) continue;
    for (int j = 0; j < n_ops; ++j)
      if (j != i && overlaps(ops[i].ptr, ops[i].bytes, ops[j].ptr, ops[j].bytes))
        return fail(B2_EINVAL, "b2_p2p: op %d (a recv) overlaps op %d", i, j);
  }
  if (const int rc = check_not_poisoned(c)) return rc;
  // Channels in order of first appearance; an op's chunks follow the chunks of the earlier ops on its channel.
  P2pArgs a{};
  int chan_peer[kP2pMaxChans];
  unsigned long long vecs = 0;
  for (int i = 0; i < n_ops; ++i) {
    const int peer = ops[i].peer, send = ops[i].is_send != 0;
    int k = 0;
    while (k < a.nchan && !(chan_peer[k] == peer && a.chan[k].send == send)) ++k;
    if (k == a.nchan) {
      const int q_me = me < peer ? me : me - 1;  // my block in the peer's arena
      const int q_peer = peer < me ? peer : peer - 1;  // the peer's block in mine
      uint8_t* recv_arena = c->arena_of[send ? peer : me] + c->p2p_off;
      uint8_t* send_arena = c->arena_of[send ? me : peer] + c->p2p_off;
      const int q_recv = send ? q_me : q_peer;  // the sender's block at the receiver
      const int q_send = send ? q_peer : q_me;  // the receiver's block at the sender
      P2pChan& ch = a.chan[a.nchan++];
      chan_peer[k] = peer;
      ch.inbox = recv_arena + 2 * p2p_lines_bytes(W) + static_cast<size_t>(q_recv) * kP2pSlots * kP2pSlotBytes;
      ch.flag = reinterpret_cast<uint32_t*>(recv_arena + static_cast<size_t>(q_recv) * kP2pSlots * kP2pLineBytes);
      ch.credit = reinterpret_cast<uint32_t*>(send_arena + p2p_lines_bytes(W) + static_cast<size_t>(q_send) * kP2pSlots * kP2pLineBytes);
      ch.count = c->p2p_counters + (send ? 0 : 8) + peer;
      ch.send = send;
      ch.nchunks = 0;
    }
    const unsigned long long nch = ops[i].bytes ? (ops[i].bytes + kP2pPayload - 1) / kP2pPayload : 1;
    P2pOp& op = a.op[i];
    op.ptr = static_cast<uint8_t*>(ops[i].ptr);
    op.bytes = ops[i].bytes;
    op.chan = static_cast<uint32_t>(k);
    op.chunk0 = a.chan[k].nchunks;
    op.nchunks = static_cast<uint32_t>(nch);
    a.chan[k].nchunks += static_cast<uint32_t>(nch);
    vecs += (ops[i].bytes + 15) / 16;
  }
  a.nops = n_ops;
  // At least one CTA per channel; the heuristic grid (or max_ctas) split evenly beyond that, and never more CTAs than chunks.
  const int per = grid_for(c, vecs, 1) / a.nchan;
  int grid = 0;
  for (int k = 0; k < a.nchan; ++k) {
    a.chan[k].cta_begin = grid;
    grid += static_cast<int>(per < 1 ? 1 : (static_cast<uint32_t>(per) < a.chan[k].nchunks ? static_cast<uint32_t>(per) : a.chan[k].nchunks));
  }
  a.done = c->p2p_counters + 32;
  a.status = c->d.status;
  a.timeout_ns = c->d.timeout_ns;
  DeviceGuard g(c->device);
  k_p2p<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "point-to-point kernel launch: %s", cudaGetErrorString(e));
  c->launches++;
  return B2_OK;
}

int b2_batchnorm_stats(b2_comm_t* c, float* mean, float* invstd, float count, size_t channels, float* running_mean,
                       float* running_var, double momentum, double eps, float* counts_out, void* stream) {
  if (channels == 0) return B2_OK;
  if (!mean || !invstd) return fail(B2_EINVAL, "b2_batchnorm_stats: null mean or invstd");
  if (!(count >= 0.0f)) return fail(B2_EINVAL, "b2_batchnorm_stats: count must be >= 0, got %g", static_cast<double>(count));
  if (!c) return fail(B2_EINVAL, "null communicator");
  const size_t row = (2 * ((channels + 3) / 4) + 1) * 16;  // mean, invstd and the count, each in whole vecs
  if (row > c->d.slice_cap)
    return fail(B2_EINVAL, "b2_batchnorm_stats: %zu channels need a %zu-byte row, a stage region holds %llu", channels, row,
                c->d.slice_cap);
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  // ATen's kernel takes eps and momentum as float parameters: the same double -> float conversion as at its launch
  k_bn_stats<<<1, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(c->d, mean, invstd, count, channels, running_mean, running_var,
                                                                    static_cast<float>(momentum), static_cast<float>(eps), counts_out);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "batchnorm stats kernel launch: %s", cudaGetErrorString(e));
  c->launches++;
  return B2_OK;
}

}  // extern "C"

namespace {

constexpr int kBnFwdUnroll = 4;  // x vecs in flight per thread (forward elementwise)
constexpr int kBnBwdUnroll = 2;  // x and dy vecs: 2 x 2 in flight per thread (backward elementwise)
constexpr int kBnStatsUnroll = 4;   // x vecs in flight per thread (forward statistics)
constexpr int kBnReduceUnroll = 2;  // x and dy vecs: 2 x 2 in flight per thread (backward reduce)

int bn_check_shape(const char* fn, int dtype, size_t M, size_t C) {
  if (dtype != B2_DT_BFLOAT16) return fail(B2_EINVAL, "%s: dtype %d is not B2_DT_BFLOAT16", fn, dtype);
  if (C == 0 || C % 8 != 0) return fail(B2_EINVAL, "%s: channels=%zu must be a positive multiple of 8", fn, C);
  if (M < 2) return fail(B2_EINVAL, "%s: rows=%zu, batch statistics need at least 2", fn, M);
  return B2_OK;
}

struct BnPtr {
  const char* name;
  const void* p;
  unsigned align;
};

int bn_check_ptrs(const char* fn, std::initializer_list<BnPtr> ps) {
  for (const BnPtr& q : ps) {
    if (!q.p) return fail(B2_EINVAL, "%s: null %s", fn, q.name);
    if (reinterpret_cast<uintptr_t>(q.p) % q.align != 0)
      return fail(B2_EINVAL, "%s: %s is not %u-byte aligned", fn, q.name, q.align);
  }
  return B2_OK;
}

// The reductions restate ATen's channels-last kernels, which ATen runs only for inputs with 32-bit indexing
// (canUse32BitIndexMath: fewer than 2^31 - 1 elements); above that ATen takes another path with other bits.
int bn_check_index32(const char* fn, size_t M, size_t C) {
  if (M > static_cast<size_t>(INT32_MAX) / C || M * C >= static_cast<size_t>(INT32_MAX))
    return fail(B2_EINVAL, "%s: rows*channels=%zu x %zu must be below 2^31 - 1 elements", fn, M, C);
  return B2_OK;
}

int bn_check_workspace(const char* fn, const void* ws, size_t have, size_t need) {
  if (need == 0) return B2_OK;
  if (!ws) return fail(B2_EINVAL, "%s: null workspace (%zu bytes needed)", fn, need);
  if (reinterpret_cast<uintptr_t>(ws) % 4 != 0) return fail(B2_EINVAL, "%s: workspace is not 4-byte aligned", fn);
  if (have < need) return fail(B2_EINVAL, "%s: workspace of %zu bytes, %zu needed", fn, have, need);
  return B2_OK;
}

}  // namespace

extern "C" {

int b2_bn_forward_elemt(const void* x, void* y, size_t rows, size_t channels, int dtype, const float* weight, const float* bias,
                        const float* mean, const float* var, double eps, float* save_invstd, int device, void* stream) {
  static const char* fn = "b2_bn_forward_elemt";
  if (const int rc = bn_check_shape(fn, dtype, rows, channels)) return rc;
  if (const int rc = bn_check_ptrs(fn, {{"x", x, 16}, {"y", y, 16}, {"weight", weight, 4}, {"bias", bias, 4}, {"mean", mean, 4},
                                        {"var", var, 4}, {"save_invstd", save_invstd, 4}}))
    return rc;
  DeviceGuard g(device);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bn::Plan p = bn::plan(rows, channels, sm_count(device), kBnFwdUnroll);
  // ATen converts eps to float at its launch (acc_t); so does this call
  k_bn2d_norm<kBnFwdUnroll><<<dim3(p.gx, p.gy), bn::kBnThreads, 0, s>>>(static_cast<const uint16_t*>(x), static_cast<uint16_t*>(y), rows,
                                                                         channels, p, mean, var, static_cast<float>(eps), save_invstd,
                                                                         weight, bias);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "batchnorm forward kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_bn_backward_elemt(const void* dy, const void* x, void* dx, size_t rows, size_t channels, int dtype, const float* weight,
                         const float* mean, const float* invstd, const float* sum_dy, const float* sum_dy_xmu, int device,
                         void* stream) {
  static const char* fn = "b2_bn_backward_elemt";
  if (const int rc = bn_check_shape(fn, dtype, rows, channels)) return rc;
  if (const int rc = bn_check_ptrs(fn, {{"dy", dy, 16}, {"x", x, 16}, {"dx", dx, 16}, {"weight", weight, 4}, {"mean", mean, 4},
                                        {"invstd", invstd, 4}, {"sum_dy", sum_dy, 4}, {"sum_dy_xmu", sum_dy_xmu, 4}}))
    return rc;
  DeviceGuard g(device);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bn::Plan p = bn::plan(rows, channels, sm_count(device), kBnBwdUnroll);
  // ATen's norm_fct: 1 / count in double, converted to float
  k_bn2d_bwd_elemt<kBnBwdUnroll><<<dim3(p.gx, p.gy), bn::kBnThreads, 0, s>>>(
      static_cast<const uint16_t*>(dy), static_cast<const uint16_t*>(x), static_cast<uint16_t*>(dx), rows, channels, p, mean, invstd,
      weight, sum_dy, sum_dy_xmu, static_cast<float>(1.0 / static_cast<double>(rows)));
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "batchnorm backward kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_bn_reduce_plan(size_t rows, size_t channels, int* geometry, size_t* workspace_bytes) {
  static const char* fn = "b2_bn_reduce_plan";
  if (const int rc = bn_check_shape(fn, B2_DT_BFLOAT16, rows, channels)) return rc;
  if (const int rc = bn_check_index32(fn, rows, channels)) return rc;
  if (!geometry || !workspace_bytes) return fail(B2_EINVAL, "%s: null geometry or workspace_bytes", fn);
  const bn::Tree t = bn::tree(static_cast<int>(rows), static_cast<int>(channels));
  geometry[0] = t.block_x;
  geometry[1] = t.block_y;
  geometry[2] = t.grid_x;
  geometry[3] = t.grid_y;
  *workspace_bytes = bn::workspace_bytes(t, static_cast<int>(channels));
  return B2_OK;
}

int b2_bn_stats(const void* x, size_t rows, size_t channels, int dtype, float* mean, float* var, float* running_mean, float* running_var,
                double momentum, void* workspace, size_t workspace_bytes, int device, void* stream) {
  static const char* fn = "b2_bn_stats";
  if (const int rc = bn_check_shape(fn, dtype, rows, channels)) return rc;
  if (const int rc = bn_check_index32(fn, rows, channels)) return rc;
  if (const int rc = bn_check_ptrs(fn, {{"x", x, 16}, {"mean", mean, 4}, {"var", var, 4}})) return rc;
  if ((running_mean == nullptr) != (running_var == nullptr))
    return fail(B2_EINVAL, "%s: running_mean and running_var must both be given or both be null", fn);
  if (running_mean)
    if (const int rc = bn_check_ptrs(fn, {{"running_mean", running_mean, 4}, {"running_var", running_var, 4}})) return rc;
  const int M = static_cast<int>(rows), C = static_cast<int>(channels);
  const bn::Tree t = bn::tree(M, C);
  if (const int rc = bn_check_workspace(fn, workspace, workspace_bytes, bn::workspace_bytes(t, C))) return rc;
  DeviceGuard g(device);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  // ATen's update lambda takes momentum as float and bessel = N / (N - 1) computed in double, rounded to float
  const float mom = static_cast<float>(momentum);
  const float bessel = static_cast<float>(static_cast<double>(rows) / static_cast<double>(rows - 1));
  float* ws = static_cast<float*>(workspace);
  const bn::ReduceGrid rg = bn::reduce_grid(t, C);
  k_bn2d_stats<kBnStatsUnroll><<<rg.grid, rg.block, 0, s>>>(static_cast<const uint16_t*>(x), M, C, t, rg.vw, mean, var, running_mean,
                                                           running_var, mom, bessel, ws);
  if (t.grid_y > 1)
    k_bn2d_stats_merge<<<rg.merge_grid, rg.merge_block, 0, s>>>(C, t, rg.mw, ws, mean, var, running_mean, running_var, mom, bessel);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "batchnorm statistics kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_bn_backward_reduce(const void* dy, const void* x, size_t rows, size_t channels, int dtype, const float* mean, const float* invstd,
                          float* sum_dy, float* sum_dy_xmu, float* grad_weight, float* grad_bias, void* workspace, size_t workspace_bytes,
                          int device, void* stream) {
  static const char* fn = "b2_bn_backward_reduce";
  if (const int rc = bn_check_shape(fn, dtype, rows, channels)) return rc;
  if (const int rc = bn_check_index32(fn, rows, channels)) return rc;
  if (const int rc = bn_check_ptrs(fn, {{"dy", dy, 16}, {"x", x, 16}, {"mean", mean, 4}, {"invstd", invstd, 4}, {"sum_dy", sum_dy, 4},
                                        {"sum_dy_xmu", sum_dy_xmu, 4}, {"grad_weight", grad_weight, 4}, {"grad_bias", grad_bias, 4}}))
    return rc;
  const int M = static_cast<int>(rows), C = static_cast<int>(channels);
  const bn::Tree t = bn::tree(M, C);
  if (const int rc = bn_check_workspace(fn, workspace, workspace_bytes, bn::workspace_bytes(t, C))) return rc;
  DeviceGuard g(device);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* ws = static_cast<float*>(workspace);
  const bn::ReduceGrid rg = bn::reduce_grid(t, C);
  k_bn2d_bwd_reduce<kBnReduceUnroll><<<rg.grid, rg.block, 0, s>>>(static_cast<const uint16_t*>(dy), static_cast<const uint16_t*>(x), M, C, t,
                                                                 rg.vw, mean, invstd, sum_dy, sum_dy_xmu, grad_weight, grad_bias, ws);
  if (t.grid_y > 1)
    k_bn2d_bwd_reduce_merge<<<rg.merge_grid, rg.merge_block, 0, s>>>(C, t, rg.mw, ws, invstd, sum_dy, sum_dy_xmu, grad_weight, grad_bias);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "batchnorm backward reduce kernel launch: %s", cudaGetErrorString(e));
  return B2_OK;
}

int b2_barrier(b2_comm_t* c, void* stream) {
  if (!c) return fail(B2_EINVAL, "null communicator");
  if (c->d.world == 1) return B2_OK;
  if (const int rc = check_not_poisoned(c)) return rc;
  DeviceGuard g(c->device);
  k_barrier<<<1, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(c->d);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B2_ECUDA, "barrier kernel launch: %s", cudaGetErrorString(e));
  c->launches++;
  return B2_OK;
}

}  // extern "C"
