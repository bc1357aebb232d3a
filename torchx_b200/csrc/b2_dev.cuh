// b2_dev.cuh — constants, the device-visible communicator view and the device helpers shared by every kernel of
// libb200ddp.so (included by b200ddp.cu only; one translation unit).
#pragma once

#include "../../include/b200ddp.h"

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

// ------------------------------------------------------------------------------------------------
// constants shared by host and device
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int kThreads = 512;                // threads per CTA for every collective kernel
constexpr int kMaxCtas = 264;                // 2 x 132 SMs (H100 SXM): upper bound on the grid of a collective
constexpr int kFlagSlotBytes = 64;           // one 64 B half-line of flags per slot (8 x u64, one per source rank)
constexpr size_t kXbarFlagBytes = 64 << 10;  // region 0: one slot per CTA index (cta_xbar: one-shot, two-shot, broadcast, barrier)
constexpr int kMaxChunks = 16;               // chunk slots per CTA index and kind in the pipeline flag region
constexpr int kPipeKinds = 2;                // X1 ("inputs staged / scattered"), X2 ("slice reduced / multicast")
constexpr size_t kPipeFlagBytes = 960 << 10;  // region 1: kMaxCtas x kPipeKinds x kMaxChunks slots; stages start 1 MiB in
constexpr size_t kFlagRegionBytes = kXbarFlagBytes + kPipeFlagBytes;
constexpr size_t kDefaultStageBytes = 512ull << 20;  // x2 stages = 1 GiB of the 80 GB: a 1 GiB fp32 bucket is one launch
// Peer waits are bounded so a dead peer can never wedge the GPU, but the bound has to be far above any legitimate
// stall of a healthy peer (rank-0 checkpoint / eval, a dataloader hiccup): NCCL's default for the same situation is 600 s.
constexpr unsigned long long kDefaultTimeoutNs = 600ull * 1000ull * 1000ull * 1000ull;

// Vecs per thread per loop trip of the multi-rank kernels: U x W wire vecs in flight per thread, without spilling
// (U*W*8 data registers).  The host sizes their grids with the same number.
__host__ __device__ constexpr int vecs_per_trip(int world) { return world >= 5 ? 1 : (world >= 3 ? 2 : (world >= 2 ? 4 : 8)); }

// "Not written yet" marker of the NVLS output buffers: a 32-bit word that reduced data never contains (as two bf16 lanes,
// as two fp16 lanes or as one fp32 it is a NaN with an all-ones payload; the producer canonicalises such a word to the
// default NaN first).
constexpr uint32_t kSentinel = 0xFFFFFFFFu;

// ---- per-mode facts --------------------------------------------------------------------------------
// Every "which mode" question the kernels and the launch code ask is answered here, so a mode that is not listed fails to
// compile instead of silently taking another mode's branch.
enum class WireFmt { kF32, kBF16, kF16 };

template <int MODE>
struct ModeTraits {
  static_assert(MODE < 0 && MODE >= 0, "unknown B2 mode: add its ModeTraits specialisation");
};
// Elem: the bucket's element type as the kernels access it (16-bit formats as raw bits); kWire: what travels between
// ranks; kCastIn: the fp32 bucket is rounded to the wire format BEFORE the scale (the hook's `.to(dtype).div_(W)`).
template <>
struct ModeTraits<B2_F32_WIRE_BF16> {
  using Elem = float;
  static constexpr int kElemBytes = 4;
  static constexpr WireFmt kWire = WireFmt::kBF16;
  static constexpr bool kCastIn = true;
};
template <>
struct ModeTraits<B2_F32> {
  using Elem = float;
  static constexpr int kElemBytes = 4;
  static constexpr WireFmt kWire = WireFmt::kF32;
  static constexpr bool kCastIn = false;
};
template <>
struct ModeTraits<B2_BF16> {
  using Elem = uint16_t;
  static constexpr int kElemBytes = 2;
  static constexpr WireFmt kWire = WireFmt::kBF16;
  static constexpr bool kCastIn = false;
};
template <>
struct ModeTraits<B2_F32_WIRE_F16> {
  using Elem = float;
  static constexpr int kElemBytes = 4;
  static constexpr WireFmt kWire = WireFmt::kF16;
  static constexpr bool kCastIn = true;
};
template <>
struct ModeTraits<B2_F16> {
  using Elem = uint16_t;
  static constexpr int kElemBytes = 2;
  static constexpr WireFmt kWire = WireFmt::kF16;
  static constexpr bool kCastIn = false;
};
template <int MODE>
constexpr bool kF32Wire = ModeTraits<MODE>::kWire == WireFmt::kF32;  // 32-byte wire vecs (else 16 bytes: 8 x 16 bit)
template <int MODE>
constexpr bool k16BitBucket = ModeTraits<MODE>::kElemBytes == 2;     // the bucket holds wire-format elements

constexpr size_t kLLFlagOff = 32 << 10;      // the LL flow-control words (8 x u64), inside region 0 past its slots
static_assert((size_t)kMaxCtas * kFlagSlotBytes <= kLLFlagOff && kLLFlagOff + kFlagSlotBytes <= kXbarFlagBytes,
              "xbar flag region too small");
static_assert((size_t)kMaxCtas * kPipeKinds * kMaxChunks * kFlagSlotBytes <= kPipeFlagBytes, "pipeline flag region too small");

// Device-visible description of one rank's view of the communicator; passed BY VALUE as a kernel
// parameter (well under the 4 KiB parameter limit), so no device-side indirection is needed.
struct CommDev {
  int rank;
  int world;
  uint8_t* peer[B2_MAX_WORLD];      // peer[jj] = symmetric arena of rank (rank + jj) % world as mapped in
                                    // THIS process (peer[0] is this rank's own).  Pre-rotated on the host so
                                    // unrolled device loops index it with compile-time constants (registers,
                                    // not a local-memory copy of the parameter block) and so the W ranks
                                    // never all target the same peer in the same loop step.
  uint8_t* mc;                      // multicast (NVLS) alias of the arena: a store to mc + off lands at arena + off on
                                    // EVERY rank, a multimem.ld_reduce from it returns the switch-side sum over all
                                    // ranks; nullptr when the fabric / driver does not expose multicast
  uint64_t* opseq;                  // local: number of collectives completed on this communicator
  uint32_t* done;                   // local: CTAs of the running collective that reached the epilogue
  uint32_t* status;                 // host-mapped: 0 = healthy, else a B2_E* code (positive)
  unsigned long long timeout_ns;    // bound on any single peer wait
  unsigned long long flag_off;      // byte offset of the cta_xbar flag region inside an arena
  unsigned long long pflag_off;     // byte offset of the pipeline flag region inside an arena
  unsigned long long stage_off[2];  // byte offsets of the two staging buffers inside an arena
  unsigned long long slice_cap;     // bytes of one region; a stage is (world + 1) regions:
                                    //   regions 0..W-1 = "recv[r]" (written by rank r), region W = "reduced";
                                    //   the NVLS path uses regions 0..W-1 as ONE contiguous message-sized buffer
  unsigned long long ll_off[2];     // per staging parity, the SENTINEL-managed buffers: 2W regions of slice_cap bytes,
                                    //   regions 0..W-1   "recv[r]"  contributions to my slice, pushed by rank r   (LL two-shot)
                                    //   regions W..2W-1  "out[j]"   reduced slice j, pushed by rank j (LL) or multicast by
                                    //                               the switch (NVLS)
                                    // Always all-SENTINEL outside a running collective: a consumer recognises arrived data
                                    // word by word as "not the sentinel" (no flag, no fence, no barrier) and puts the
                                    // sentinel back after reading.
  unsigned long long llflag_off;    // 8 x u64: llflag[r] = op counter of the latest LL collective rank r has STARTED
                                    // (flow control: nobody writes a parity's buffers before their owner has left the
                                    // collective that last used them)
  unsigned long long* trace;        // optional (b2_comm_trace): per-CTA globaltimer stamps of the LAST collective,
                                    // 8 slots per CTA (see include/b200ddp.h)
};

// Where a collective reads its INPUT from.  nseg == 0: the bucket itself (in place).  Otherwise the bucket is only the
// OUTPUT and the input is gathered straight from the per-parameter gradient tensors ("zero-copy bucket fill": the
// Reducer's copy-in pass, torch/csrc/distributed/c10d/reducer.cpp mark_variable_ready_dense, disappears into the first
// phase of the allreduce): segment i holds bucket elements [begin[i], begin[i+1]) at ptr[i], in bucket order and without
// gaps.  The table travels BY VALUE in the kernel parameters (constant bank: ~2 KiB of the 4 KiB limit) - no device-side
// table, no host-to-device copy to order against the launch, nothing to keep alive.
constexpr int kMaxSegs = B2_MAX_SEGMENTS;
struct Src {
  int nseg;
  unsigned long long off;  // bucket element index of this launch's element 0 (messages larger than a stage are cut up)
  const void* ptr[kMaxSegs];
  unsigned long long begin[kMaxSegs + 1];
};

}  // namespace

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
namespace dev {

struct F8 {
  float v[8];
};

// An 8-float vec as the two 16-byte words it travels in, and back (bit casts, no arithmetic).
__device__ __forceinline__ void f8_to_u4(const F8& f, uint4& a, uint4& b) {
  a = make_uint4(__float_as_uint(f.v[0]), __float_as_uint(f.v[1]), __float_as_uint(f.v[2]), __float_as_uint(f.v[3]));
  b = make_uint4(__float_as_uint(f.v[4]), __float_as_uint(f.v[5]), __float_as_uint(f.v[6]), __float_as_uint(f.v[7]));
}
__device__ __forceinline__ F8 f8_from_u4(const uint4& a, const uint4& b) {
  return F8{{__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(a.w),
             __uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(b.w)}};
}

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t ld_volatile_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// 128-bit streaming accesses (LDG.E.128 / STG.E.128).  Hopper has no 256-bit global load or store, so an 8-float vec is
// two of them, both issued before either result is used.
__device__ __forceinline__ F8 ldg_f8(const float* p) {
  F8 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3])
               : "l"(p)
               : "memory");
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.v[4]), "=f"(r.v[5]), "=f"(r.v[6]), "=f"(r.v[7])
               : "l"(p + 4)
               : "memory");
  return r;
}
__device__ __forceinline__ void stg_f8(float* p, const F8& r) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(r.v[0]), "f"(r.v[1]),
               "f"(r.v[2]), "f"(r.v[3])
               : "memory");
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + 4), "f"(r.v[4]), "f"(r.v[5]),
               "f"(r.v[6]), "f"(r.v[7])
               : "memory");
}
__device__ __forceinline__ uint4 ldg_u4(const void* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void stg_u4(void* p, const uint4& r) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(r.x), "r"(r.y),
               "r"(r.z), "r"(r.w)
               : "memory");
}

// ---- NVLS (NVSwitch multicast) accesses ----------------------------------------------------------
// `p` is an address inside the MULTICAST mapping of the arena.  ld_reduce: the switch reads the 16 bytes at this
// offset from every rank's arena, adds them (bf16x2 lanes, fp32 accumulation inside the switch, one rounding back
// to bf16) and returns one result - (W-1)/W of the reduce-scatter traffic never enters this GPU.  st: the switch
// replicates the 16 bytes into every rank's arena - the all-gather leaves this GPU once instead of W-1 times.
// SASS: MULTIMEM.LD_REDUCE / MULTIMEM.ST.
__device__ __forceinline__ uint4 mm_ld_reduce_bf16x2(const void* p) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
// The same with f16x2 lanes (SASS LDGMC.E.F32ADD.F16x8.RN): fp32 accumulation inside the switch, one rounding to fp16.
__device__ __forceinline__ uint4 mm_ld_reduce_f16x2(const void* p) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ uint4 mm_ld_reduce_f32(const void* p) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void mm_st_u4(void* p, const uint4& r) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(r.x), "r"(r.y), "r"(r.z),
               "r"(r.w)
               : "memory");
}

// 16-byte load that always goes to L2 (polling for data another GPU / the switch writes): LDG.E.128.STRONG.SYS
__device__ __forceinline__ uint4 ld_volatile_u4(const void* p) {
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ bool has_sentinel(const uint4& q) {
  return q.x == kSentinel || q.y == kSentinel || q.z == kSentinel || q.w == kSentinel;
}
// reduced data never carries the sentinel: an all-ones NaN word becomes the default NaN (bf16x2 / f16x2: both lanes;
// 0x7FFF is a quiet NaN in both 16-bit formats)
template <bool F32>
__device__ __forceinline__ uint4 no_sentinel(uint4 q) {
  constexpr uint32_t kNan = F32 ? 0x7FFFFFFFu : 0x7FFF7FFFu;
  if (q.x == kSentinel) q.x = kNan;
  if (q.y == kSentinel) q.y = kNan;
  if (q.z == kSentinel) q.z = kNan;
  if (q.w == kSentinel) q.w = kNan;
  return q;
}

// fp32 pair -> packed bf16x2 with round-to-nearest-even (one F2FP.BF16.F32.PACK_AB). `lo` lands
// in bits [15:0] (the lower address in little-endian memory), `hi` in bits [31:16].
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float bf16_lo(uint32_t p) { return __uint_as_float(p << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t p) { return __uint_as_float(p & 0xffff0000u); }

// fp32 pair -> packed f16x2, IEEE round-to-nearest-even (F2FP.F16.F32.PACK_AB).  Subnormals are kept, overflow gives
// +-inf (no .satfinite: an overflowed scaled gradient must stay inf), NaN gives a NaN.  Lane order as pack_bf16x2.
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// fp16 -> fp32 is exact (every fp16 value, subnormals included, is an fp32 normal).
__device__ __forceinline__ float f16_to_f32(uint16_t h) {
  float f;
  asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
  return f;
}
__device__ __forceinline__ float f16_lo(uint32_t p) { return f16_to_f32(static_cast<uint16_t>(p & 0xffffu)); }
__device__ __forceinline__ float f16_hi(uint32_t p) { return f16_to_f32(static_cast<uint16_t>(p >> 16)); }

// The 16-bit wire formats, selected by mode: pack two fp32 into one word (the rounding), widen either lane (exact).
template <int MODE>
__device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  static_assert(!kF32Wire<MODE>, "pack16: 16-bit wire modes only");
  if constexpr (ModeTraits<MODE>::kWire == WireFmt::kF16) return pack_f16x2(lo, hi);
  else return pack_bf16x2(lo, hi);
}
template <int MODE>
__device__ __forceinline__ float lo16(uint32_t p) {
  if constexpr (ModeTraits<MODE>::kWire == WireFmt::kF16) return f16_lo(p);
  else return bf16_lo(p);
}
template <int MODE>
__device__ __forceinline__ float hi16(uint32_t p) {
  if constexpr (ModeTraits<MODE>::kWire == WireFmt::kF16) return f16_hi(p);
  else return bf16_hi(p);
}
// One bucket element (as ModeTraits<MODE>::Elem) -> fp32.
template <int MODE>
__device__ __forceinline__ float elem_to_f32(typename ModeTraits<MODE>::Elem x) {
  if constexpr (k16BitBucket<MODE>) return lo16<MODE>(static_cast<uint32_t>(x));
  else return x;
}

// ---- wire vecs -----------------------------------------------------------------------------------
// A "vec" is 8 consecutive elements everywhere in this library.
template <int MODE, bool F32 = kF32Wire<MODE>>
struct Wire;  // wire representation of one vec

template <int MODE>
struct Wire<MODE, false> {  // 8 x 16 bit: bf16x2 or f16x2 words
  static constexpr int kBytes = 16;
  uint4 q;
};
template <int MODE>
struct Wire<MODE, true> {  // 8 x fp32
  static constexpr int kBytes = 32;
  F8 f;
};

template <int MODE>
__device__ __forceinline__ Wire<MODE> ld_wire(const uint8_t* p) {
  Wire<MODE> w;
  if constexpr (kF32Wire<MODE>) {
    w.f = ldg_f8(reinterpret_cast<const float*>(p));
  } else {
    w.q = ldg_u4(p);
  }
  return w;
}
template <int MODE>
__device__ __forceinline__ void st_wire(uint8_t* p, const Wire<MODE>& w) {
  if constexpr (kF32Wire<MODE>) {
    stg_f8(reinterpret_cast<float*>(p), w.f);
  } else {
    stg_u4(p, w.q);
  }
}

// switch-side sum of one wire vec over all ranks / replicated store of one wire vec to all ranks
template <int MODE>
__device__ __forceinline__ Wire<MODE> mm_ld_reduce_wire(const uint8_t* p) {
  Wire<MODE> w;
  if constexpr (kF32Wire<MODE>) {
    const uint4 a = mm_ld_reduce_f32(p), b = mm_ld_reduce_f32(p + 16);
    w.f = f8_from_u4(a, b);
  } else if constexpr (ModeTraits<MODE>::kWire == WireFmt::kF16) {
    w.q = mm_ld_reduce_f16x2(p);
  } else {
    w.q = mm_ld_reduce_bf16x2(p);
  }
  return w;
}
template <int MODE>
__device__ __forceinline__ void mm_st_wire(uint8_t* p, const Wire<MODE>& w) {
  if constexpr (kF32Wire<MODE>) {
    uint4 a, b;
    f8_to_u4(w.f, a, b);
    mm_st_u4(p, a);
    mm_st_u4(p + 16, b);
  } else {
    mm_st_u4(p, w.q);
  }
}

// ---- sentinel protocol of the NVLS output buffer (see CommDev::nvls_out_off) -----------------------------------------
template <int MODE>
__device__ __forceinline__ Wire<MODE> wire_no_sentinel(Wire<MODE> w) {
  if constexpr (kF32Wire<MODE>) {
    uint4 a, b;
    f8_to_u4(w.f, a, b);
    w.f = f8_from_u4(no_sentinel<true>(a), no_sentinel<true>(b));
  } else {
    w.q = no_sentinel<false>(w.q);
  }
  return w;
}
// One poll of a wire vec in the output buffer; `pending` = some 32-bit word still holds the sentinel (a 16-byte multicast
// store lands as a whole, but every word is checked anyway).
template <int MODE>
__device__ __forceinline__ Wire<MODE> wire_poll(const uint8_t* p, bool* pending) {
  Wire<MODE> w;
  if constexpr (kF32Wire<MODE>) {
    const uint4 a = ld_volatile_u4(p), b = ld_volatile_u4(p + 16);
    *pending = has_sentinel(a) || has_sentinel(b);
    w.f = f8_from_u4(a, b);
  } else {
    w.q = ld_volatile_u4(p);
    *pending = has_sentinel(w.q);
  }
  return w;
}
template <int MODE>
__device__ __forceinline__ void wire_reset(uint8_t* p) {
  const uint4 s4 = make_uint4(kSentinel, kSentinel, kSentinel, kSentinel);
  stg_u4(p, s4);
  if constexpr (kF32Wire<MODE>) stg_u4(p + 16, s4);
}

// wire(scale * x): the value a rank contributes.  Rounding points are part of the contract
// (oracle/allreduce_oracle.c: b2o_compress):
//   F32_WIRE_BF16 : bf16( float(bf16(x)) * scale )      == `buf.to(bf16).div_(W)` for W = 2^k
//   BF16          : bf16( float(x) * scale )            (x is already bf16)
//   F32           : x * scale                           == Reducer's `mul_out(bucket, grad, 1/W)`
//   F32_WIRE_F16  : f16( float(f16(x)) * scale )        == `buf.to(fp16).div_(W)` (fp16_compress_hook)
//   F16           : f16( float(x) * scale )             (x is already fp16)
template <int MODE>
__device__ __forceinline__ Wire<MODE> compress(const F8& x, float scale) {
  Wire<MODE> w;
  if constexpr (kF32Wire<MODE>) {
#pragma unroll
    for (int i = 0; i < 8; ++i) w.f.v[i] = __fmul_rn(x.v[i], scale);
  } else {
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float a = x.v[2 * i], b = x.v[2 * i + 1];
      if constexpr (ModeTraits<MODE>::kCastIn) {
        const uint32_t p = pack16<MODE>(a, b);  // first rounding: the `.to(bf16 / fp16)` cast
        a = lo16<MODE>(p);
        b = hi16<MODE>(p);
      }
      o[i] = pack16<MODE>(__fmul_rn(a, scale), __fmul_rn(b, scale));
    }
    w.q = make_uint4(o[0], o[1], o[2], o[3]);
  }
  return w;
}

template <int MODE>
__device__ __forceinline__ F8 widen(const Wire<MODE>& w) {
  if constexpr (kF32Wire<MODE>) {
    return w.f;
  } else {
    F8 r;
    r.v[0] = lo16<MODE>(w.q.x);
    r.v[1] = hi16<MODE>(w.q.x);
    r.v[2] = lo16<MODE>(w.q.y);
    r.v[3] = hi16<MODE>(w.q.y);
    r.v[4] = lo16<MODE>(w.q.z);
    r.v[5] = hi16<MODE>(w.q.z);
    r.v[6] = lo16<MODE>(w.q.w);
    r.v[7] = hi16<MODE>(w.q.w);
    return r;
  }
}

// round(s): the reduced value as it travels in the gather phase / is stored.
template <int MODE>
__device__ __forceinline__ Wire<MODE> finalize(const F8& s) {
  Wire<MODE> w;
  if constexpr (kF32Wire<MODE>) {
    w.f = s;
  } else {
    w.q = make_uint4(pack16<MODE>(s.v[0], s.v[1]), pack16<MODE>(s.v[2], s.v[3]),
                     pack16<MODE>(s.v[4], s.v[5]), pack16<MODE>(s.v[6], s.v[7]));
  }
  return w;
}

__device__ __forceinline__ void accumulate(F8& s, const F8& c) {
#pragma unroll
  for (int i = 0; i < 8; ++i) s.v[i] = __fadd_rn(s.v[i], c.v[i]);
}

// The W contributions to one vec summed in rank order, in fp32 (oracle/allreduce_oracle.c: b2o_allreduce).  k_twoshot and
// k_pipe take the sum in a statement of its own before the store: as an argument of st_wire it reorders their SASS.
template <int MODE, int W>
__device__ __forceinline__ F8 reduce_rank_order(const Wire<MODE> (&w)[W]) {
  F8 s = widen<MODE>(w[0]);
#pragma unroll
  for (int r = 1; r < W; ++r) accumulate(s, widen<MODE>(w[r]));
  return s;
}

// ---- local bucket accesses (the caller's tensor: any alignment, any length) --------------------
template <int MODE>
__device__ __forceinline__ F8 load_in(const void* buf, unsigned long long e, unsigned long long n,
                                      bool aligned) {
  F8 x;
  if constexpr (k16BitBucket<MODE>) {  // the bucket holds wire-format elements
    const uint16_t* p = reinterpret_cast<const uint16_t*>(buf) + e;
    if (aligned && e + 8 <= n) {
      Wire<MODE> w;
      w.q = ldg_u4(p);
      x = widen<MODE>(w);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        x.v[i] = (e + i < n) ? elem_to_f32<MODE>(p[i]) : 0.f;
    }
  } else {
    const float* p = reinterpret_cast<const float*>(buf) + e;
    if (aligned && e + 8 <= n) {
      x = ldg_f8(p);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) x.v[i] = (e + i < n) ? p[i] : 0.f;
    }
  }
  return x;
}

// `w` is the reduced vec in wire format; writes it to the caller's tensor in the tensor's dtype.
template <int MODE>
__device__ __forceinline__ void store_out(void* buf, unsigned long long e, unsigned long long n,
                                          bool aligned, const Wire<MODE>& w) {
  if constexpr (k16BitBucket<MODE>) {  // the wire bits are the bucket's bits
    uint16_t* p = reinterpret_cast<uint16_t*>(buf) + e;
    if (aligned && e + 8 <= n) {
      stg_u4(p, w.q);
    } else {
      const uint32_t q[4] = {w.q.x, w.q.y, w.q.z, w.q.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (e + i < n) p[i] = static_cast<uint16_t>((q[i >> 1] >> ((i & 1) * 16)) & 0xffffu);
    }
  } else {
    float* p = reinterpret_cast<float*>(buf) + e;
    const F8 r = widen<MODE>(w);
    if (aligned && e + 8 <= n) {
      stg_f8(p, r);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (e + i < n) p[i] = r.v[i];
    }
  }
}

template <int MODE>
__device__ __forceinline__ bool buf_aligned(const void* buf) {
  return (reinterpret_cast<uintptr_t>(buf) & (8u * ModeTraits<MODE>::kElemBytes - 1u)) == 0;  // one vec: 16 or 32 bytes
}

// One input vec (elements [e, e + 8) of this launch) from wherever `src` says the input lives.
// The segment a thread found last: consecutive vecs of one thread usually fall into the same parameter, so the binary
// search over the table (dependent constant-bank loads in front of the data load) is skipped most of the time.
struct SegHint {
  int s = 0;
  unsigned long long sb = 1, se = 0;  // empty range: the first lookup searches
};

template <int MODE>
__device__ __forceinline__ F8 load_src(const Src& src, SegHint& hint, const void* buf, unsigned long long e,
                                       unsigned long long n, bool aligned) {
  if (src.nseg == 0) return load_in<MODE>(buf, e, n, aligned);
  using Elem = typename ModeTraits<MODE>::Elem;
  const unsigned long long ge = e + src.off;  // bucket coordinates
  int s = hint.s;
  unsigned long long sb = hint.sb, se = hint.se;
  if (ge < sb || ge >= se) {                  // not in the segment this thread looked at last: binary search
    int lo = 0, hi = src.nseg;                // begin[lo] <= ge < begin[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (ge >= src.begin[mid]) lo = mid;
      else hi = mid;
    }
    s = lo;
    sb = src.begin[s];
    se = src.begin[s + 1];
    hint.s = s;
    hint.sb = sb;
    hint.se = se;
  }
  // A null pointer is a zero segment (B2_SEGMENT_ZEROS): its elements read as +0.0 without a load.  The address is formed
  // as an integer so that a zero segment never becomes arithmetic on a null pointer.
  const Elem* base = static_cast<const Elem*>(src.ptr[s]);
  const uintptr_t a = reinterpret_cast<uintptr_t>(base) + (ge - sb) * sizeof(Elem);
  F8 x = {};
  if (e + 8 <= n && ge + 8 <= se && (a & (8u * sizeof(Elem) - 1u)) == 0) {
    if (base) {
      const Elem* p = reinterpret_cast<const Elem*>(a);
      if constexpr (k16BitBucket<MODE>) {
        Wire<MODE> w;
        w.q = ldg_u4(p);
        x = widen<MODE>(w);
      } else {
        x = ldg_f8(p);
      }
    }
  } else {  // the vec straddles parameters, is not 32 B-aligned in its tensor, or is the ragged tail
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = 0.f;
      if (e + i < n) {
        const unsigned long long g = ge + i;
        while (g >= se) {
          ++s;
          sb = se;
          se = src.begin[s + 1];
          base = static_cast<const Elem*>(src.ptr[s]);
        }
        if (base) v = elem_to_f32<MODE>(base[g - sb]);
      }
      x.v[i] = v;
    }
  }
  return x;
}

// Without a hint (the multi-rank kernels: the W slices one thread touches are far apart, a hint would only cost registers).
template <int MODE>
__device__ __forceinline__ F8 load_src(const Src& src, const void* buf, unsigned long long e, unsigned long long n, bool aligned) {
  SegHint none;
  return load_src<MODE>(src, none, buf, e, n, aligned);
}

// peer[jj] for a RUNTIME jj without putting the parameter block into local memory (select chain)
__device__ __forceinline__ uint8_t* peer_sel(const CommDev& c, int jj) {
  uint8_t* a = c.peer[0];
#pragma unroll
  for (int i = 1; i < B2_MAX_WORLD; ++i)
    if (jj == i) a = c.peer[i];
  return a;
}

// Rank whose slice a rank visits jj-th (jj < 2W): (rank + jj) mod W, the order peer[] is rotated in.
template <int W>
__device__ __forceinline__ int slice_of(int rank, int jj) {
  int j = rank + jj;
  if (j >= W) j -= W;
  return j;
}

// slice_of for the kernels that take the world size at run time (jj < W).
__device__ __forceinline__ int rank_at(const CommDev& c, int jj) {
  int r = c.rank + jj;
  if (r >= c.world) r -= c.world;
  return r;
}

// Record B2_E* `code` in the host-mapped status word (b2_comm_status): B2_ETIMEOUT when a peer wait gave up (results are
// undefined from here on, but the GPU is not hung), B2_EINVAL when ranks disagreed on sizes.
__device__ __forceinline__ void record_status(uint32_t* status, int code) {
  *reinterpret_cast<volatile uint32_t*>(status) = static_cast<uint32_t>(-code);
  __threadfence_system();
}

// Bounded wait until *flag >= seq.  Flags and sequence numbers are 64-bit and only grow (one op per increment never
// wraps), so a plain unsigned compare is exact: a never-written (0) or stale slot is always behind.  Polls with
// ld.acquire.sys itself rather than relaxed polling + one fence.acq_rel.sys at the end: the standalone fence is a full
// MEMBAR.SYS that also drains this SM's outstanding stores, the acquire load is not.
__device__ __forceinline__ void wait_flag(const CommDev& c, const uint64_t* flag, uint64_t seq) {
  unsigned long long t0 = 0;
  unsigned spins = 0;
  while (ld_acquire_sys(flag) < seq) {
    if ((++spins & 63u) == 0) {
      const unsigned long long now = globaltimer_ns();
      if (t0 == 0) {
        t0 = now;
      } else if (now - t0 > c.timeout_ns) {
        record_status(c.status, B2_ETIMEOUT);
        break;
      }
    }
  }
}

// Poll one wire vec until no word holds the sentinel, sleeping kSleepNs between polls and reading the clock every
// kClockEvery (a power of two) polls; bounded like every other wait.
template <int MODE, unsigned kSleepNs, unsigned kClockEvery>
__device__ __forceinline__ void wait_wire(const CommDev& c, const uint8_t* p, Wire<MODE>& w) {
  static_assert((kClockEvery & (kClockEvery - 1u)) == 0, "kClockEvery must be a power of two");
  unsigned long long t0 = 0;
  unsigned spins = 0;
  bool pending = true;
  while (pending) {
    __nanosleep(kSleepNs);
    w = wire_poll<MODE>(p, &pending);
    if (pending && (++spins & (kClockEvery - 1u)) == 0) {
      const unsigned long long now = globaltimer_ns();
      if (t0 == 0) {
        t0 = now;
      } else if (now - t0 > c.timeout_ns) {
        record_status(c.status, B2_ETIMEOUT);
        break;
      }
    }
  }
}

// ---- cross-GPU barrier among the CTAs with the same blockIdx.x on every rank --------------------
// Thread p (< world) publishes `seq` into peer p's flag slot for this CTA index and waits for peer
// p's `seq` in its own slot.  Sequence numbers only grow, so "flag >= seq" is the test.
__device__ __forceinline__ void cta_xbar(const CommDev& c, uint64_t seq) {
  __syncthreads();  // all of this CTA's data stores are ordered before the release below
  if (threadIdx.x < c.world) {
    const int jj = threadIdx.x;  // this thread pairs with rank p = (rank + jj) % world
    const int p = rank_at(c, jj);
    const size_t slot = c.flag_off + static_cast<size_t>(blockIdx.x) * kFlagSlotBytes;
    uint64_t* theirs = reinterpret_cast<uint64_t*>(peer_sel(c, jj) + slot) + c.rank;
    const uint64_t* mine = reinterpret_cast<const uint64_t*>(c.peer[0] + slot) + p;
    st_release_sys(theirs, seq);
    wait_flag(c, mine, seq);
  }
  __syncthreads();  // peers' data is now visible to every thread of this CTA
}

// Every collective kernel starts by reading the communicator's op counter (parity selects the
// staging buffer, the value seeds this op's flag sequence numbers) and ends by bumping it once
// all CTAs are through.  Keeping the counter on the device makes the launch sequence CUDA-graph
// replayable and keeps the host stateless.  The bump is an add, not a store of seq0 + 1 (nothing else
// writes the counter while a collective runs): the 64-bit seq0 need not stay live to the end of the kernel.
__device__ __forceinline__ uint64_t op_begin(const CommDev& c) { return ld_volatile_u64(c.opseq); }

// The staging buffer of the op whose counter is seq0: consecutive ops alternate between the two.
__device__ __forceinline__ unsigned long long stage_of(const CommDev& c, uint64_t seq0) {
  return (seq0 & 1u) ? c.stage_off[1] : c.stage_off[0];
}

__device__ __forceinline__ void op_end(const CommDev& c) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(c.done, 1u) == gridDim.x - 1) {
      *reinterpret_cast<volatile uint32_t*>(c.done) = 0;
      __threadfence();
      atomicAdd(reinterpret_cast<unsigned long long*>(c.opseq), 1ull);
    }
  }
}

__device__ __forceinline__ void trace_stamp(const CommDev& c, int slot) {
  if (c.trace != nullptr) c.trace[blockIdx.x * 8 + slot] = globaltimer_ns();
}

}  // namespace dev
