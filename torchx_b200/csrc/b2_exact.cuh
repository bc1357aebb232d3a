// b2_exact.cuh — the exact collectives: integer SUM and MIN / MAX allreduce (b2_allreduce_op) and all-gather
// (b2_allgather).  Both are one-shot and sized for latency: every rank pushes its raw message as 16-byte vecs into
// recv[me] of every rank's stage, one cta_xbar, then each rank reads the W copies out of its own stage.  Nothing is
// rounded or converted on the way, so the result is the same bits on every rank.
//
// The stage is always addressed in vecs (it is aligned on every rank), so CTA b of every rank touches the same stage bytes
// whatever the alignment of its own buffers; only the local side falls back to element accesses, for a buffer that is not
// 16 B-aligned and for the vec that holds the end of the message.  The op counter, stage parity and flag sequence are
// those of every other collective, so these kernels interleave freely with allreduces, broadcasts and barriers.
#pragma once

#include "b2_dev.cuh"

namespace exact {

// Name (as torch spells it), element size and kind of each B2_DT_* (include/b200ddp.h).
template <int DT>
struct DtypeTraits {
  static_assert(DT < 0 && DT >= 0, "unknown B2 dtype: add its DtypeTraits specialisation");
};
template <>
struct DtypeTraits<B2_DT_INT32> {
  static constexpr const char* kName = "int32";
  static constexpr int kBytes = 4;
  static constexpr bool kInt = true;
};
template <>
struct DtypeTraits<B2_DT_INT64> {
  static constexpr const char* kName = "int64";
  static constexpr int kBytes = 8;
  static constexpr bool kInt = true;
};
template <>
struct DtypeTraits<B2_DT_FLOAT32> {
  static constexpr const char* kName = "float32";
  static constexpr int kBytes = 4;
  static constexpr bool kInt = false;
};
template <>
struct DtypeTraits<B2_DT_BFLOAT16> {
  static constexpr const char* kName = "bfloat16";
  static constexpr int kBytes = 2;
  static constexpr bool kInt = false;
};
template <>
struct DtypeTraits<B2_DT_FLOAT16> {
  static constexpr const char* kName = "float16";
  static constexpr int kBytes = 2;
  static constexpr bool kInt = false;
};

// The float MIN / MAX use the .NaN forms: a NaN in either input gives the canonical NaN, and +0.0 > -0.0 (IEEE 754-2019
// minimum / maximum).  No .ftz: subnormals are ordinary values.
__device__ __forceinline__ uint32_t min_f32(uint32_t a, uint32_t b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(__uint_as_float(a)), "f"(__uint_as_float(b)));
  return __float_as_uint(r);
}
__device__ __forceinline__ uint32_t max_f32(uint32_t a, uint32_t b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(__uint_as_float(a)), "f"(__uint_as_float(b)));
  return __float_as_uint(r);
}
__device__ __forceinline__ uint32_t min_bf16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("min.NaN.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}
__device__ __forceinline__ uint32_t max_bf16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("max.NaN.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}
__device__ __forceinline__ uint32_t min_f16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("min.NaN.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}
__device__ __forceinline__ uint32_t max_f16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("max.NaN.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

// One 32-bit word of a vec: one int32 / fp32 element or two 16-bit elements.
template <int DT, int OP>
__device__ __forceinline__ uint32_t combine32(uint32_t a, uint32_t b) {
  if constexpr (DT == B2_DT_INT32) {
    if constexpr (OP == B2_OP_SUM) return a + b;  // two's complement: wraps modulo 2^32
    else if constexpr (OP == B2_OP_MIN) return static_cast<uint32_t>(min(static_cast<int32_t>(a), static_cast<int32_t>(b)));
    else return static_cast<uint32_t>(max(static_cast<int32_t>(a), static_cast<int32_t>(b)));
  } else if constexpr (DT == B2_DT_FLOAT32) {
    static_assert(OP != B2_OP_SUM, "float SUM runs on the rank-order allreduce kernels");
    return OP == B2_OP_MIN ? min_f32(a, b) : max_f32(a, b);
  } else if constexpr (DT == B2_DT_BFLOAT16) {
    static_assert(OP != B2_OP_SUM, "float SUM runs on the rank-order allreduce kernels");
    return OP == B2_OP_MIN ? min_bf16x2(a, b) : max_bf16x2(a, b);
  } else {
    static_assert(DT == B2_DT_FLOAT16 && OP != B2_OP_SUM, "float SUM runs on the rank-order allreduce kernels");
    return OP == B2_OP_MIN ? min_f16x2(a, b) : max_f16x2(a, b);
  }
}

// One 64-bit element held in two words (little-endian: lo first).
template <int OP>
__device__ __forceinline__ void combine64(uint32_t& lo, uint32_t& hi, uint32_t blo, uint32_t bhi) {
  const long long a = static_cast<long long>((static_cast<unsigned long long>(hi) << 32) | lo);
  const long long b = static_cast<long long>((static_cast<unsigned long long>(bhi) << 32) | blo);
  unsigned long long r;
  if constexpr (OP == B2_OP_SUM) r = static_cast<unsigned long long>(a) + static_cast<unsigned long long>(b);  // wraps mod 2^64
  else if constexpr (OP == B2_OP_MIN) r = static_cast<unsigned long long>(a < b ? a : b);
  else r = static_cast<unsigned long long>(a < b ? b : a);
  lo = static_cast<uint32_t>(r);
  hi = static_cast<uint32_t>(r >> 32);
}

template <int DT, int OP>
__device__ __forceinline__ uint4 combine(uint4 a, const uint4& b) {
  if constexpr (DT == B2_DT_INT64) {
    combine64<OP>(a.x, a.y, b.x, b.y);
    combine64<OP>(a.z, a.w, b.z, b.w);
  } else {
    a.x = combine32<DT, OP>(a.x, b.x);
    a.y = combine32<DT, OP>(a.y, b.y);
    a.z = combine32<DT, OP>(a.z, b.z);
    a.w = combine32<DT, OP>(a.w, b.w);
  }
  return a;
}

// Vec v of a message of n elements of E bytes at `p`, element by element: elements at or past n read as zero.  For a
// buffer that is not 16 B-aligned (it is always E-aligned) and for the vec that holds the end of the message.
template <int E>
__device__ __forceinline__ uint4 ld_elems(const uint8_t* p, unsigned long long v, unsigned long long n) {
  constexpr int kPer = 16 / E;
  uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    const unsigned long long e = v * kPer + i;
    if (e < n) {
      if constexpr (E == 8) {
        const unsigned long long x = reinterpret_cast<const unsigned long long*>(p)[e];
        w[2 * i] = static_cast<uint32_t>(x);
        w[2 * i + 1] = static_cast<uint32_t>(x >> 32);
      } else if constexpr (E == 4) {
        w[i] = reinterpret_cast<const uint32_t*>(p)[e];
      } else if constexpr (E == 2) {
        w[i >> 1] |= static_cast<uint32_t>(reinterpret_cast<const uint16_t*>(p)[e]) << ((i & 1) * 16);
      } else {
        w[i >> 2] |= static_cast<uint32_t>(p[e]) << ((i & 3) * 8);
      }
    }
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// The store twin of ld_elems: writes only the elements of vec v that are below n.
template <int E>
__device__ __forceinline__ void st_elems(uint8_t* p, unsigned long long v, unsigned long long n, const uint4& q) {
  constexpr int kPer = 16 / E;
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    const unsigned long long e = v * kPer + i;
    if (e < n) {
      if constexpr (E == 8) {
        reinterpret_cast<unsigned long long*>(p)[e] =
            (static_cast<unsigned long long>(w[2 * i + 1]) << 32) | w[2 * i];
      } else if constexpr (E == 4) {
        reinterpret_cast<uint32_t*>(p)[e] = w[i];
      } else if constexpr (E == 2) {
        reinterpret_cast<uint16_t*>(p)[e] = static_cast<uint16_t>(w[i >> 1] >> ((i & 1) * 16));
      } else {
        p[e] = static_cast<uint8_t>(w[i >> 2] >> ((i & 3) * 8));
      }
    }
  }
}

// Vec v of this rank's message: one 16-byte load when it lies wholly inside an aligned buffer.
template <int E>
__device__ __forceinline__ uint4 ld_local(const uint8_t* p, bool aligned, unsigned long long v, unsigned long long n) {
  if (aligned && (v + 1) * (16 / E) <= n) return dev::ldg_u4(p + v * 16);
  return ld_elems<E>(p, v, n);
}

template <int E>
__device__ __forceinline__ void st_local(uint8_t* p, bool aligned, unsigned long long v, unsigned long long n, const uint4& q) {
  if (aligned && (v + 1) * (16 / E) <= n) dev::stg_u4(p + v * 16, q);
  else st_elems<E>(p, v, n, q);
}

// Push vec v of my message into recv[me] of every rank (mine included).
__device__ __forceinline__ void push_vec(const CommDev& c, unsigned long long stage, unsigned long long v, const uint4& q) {
#pragma unroll
  for (int jj = 0; jj < B2_MAX_WORLD; ++jj)
    if (jj < c.world) dev::stg_u4(c.peer[jj] + stage + c.rank * c.slice_cap + v * 16, q);
}

}  // namespace exact

// buf[i] <- OP over r of buf_r[i], combined in rank order.  n elements; a launch holds at most slice_cap bytes.
template <int DT, int OP>
__global__ void __launch_bounds__(kThreads, 1) k_reduce_exact(CommDev c, void* buf, unsigned long long n) {
  using namespace dev;
  constexpr int E = exact::DtypeTraits<DT>::kBytes;
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  uint8_t* p = static_cast<uint8_t*>(buf);
  const bool aligned = (reinterpret_cast<uintptr_t>(buf) & 15u) == 0;
  const unsigned long long V = (n * E + 15) / 16;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  for (unsigned long long v = first; v < V; v += stride) exact::push_vec(c, stage, v, exact::ld_local<E>(p, aligned, v, n));
  cta_xbar(c, seq0 * 4u + 1u);
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

// Rank r's `bytes` bytes land at out + r * block.  `in` may be this rank's own block (torch's in-place form): that block
// is then left alone.  A launch holds at most slice_cap bytes per rank.
__global__ void __launch_bounds__(kThreads, 1)
    k_allgather(CommDev c, uint8_t* out, const uint8_t* in, unsigned long long bytes, unsigned long long block) {
  using namespace dev;
  const uint64_t seq0 = op_begin(c);
  const unsigned long long stage = stage_of(c, seq0);
  const bool in_aligned = (reinterpret_cast<uintptr_t>(in) & 15u) == 0;
  const bool in_place = in == out + static_cast<unsigned long long>(c.rank) * block;
  const unsigned long long V = (bytes + 15) / 16;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  for (unsigned long long v = first; v < V; v += stride) exact::push_vec(c, stage, v, exact::ld_local<1>(in, in_aligned, v, bytes));
  cta_xbar(c, seq0 * 4u + 1u);
  const uint8_t* mine = c.peer[0] + stage;
  for (unsigned long long v = first; v < V; v += stride) {
    uint4 q[B2_MAX_WORLD];
#pragma unroll
    for (int r = 0; r < B2_MAX_WORLD; ++r)
      if (r < c.world) q[r] = ldg_u4(mine + r * c.slice_cap + v * 16);
#pragma unroll
    for (int r = 0; r < B2_MAX_WORLD; ++r) {
      if (r < c.world && !(in_place && r == c.rank)) {
        uint8_t* dst = out + static_cast<unsigned long long>(r) * block;
        exact::st_local<1>(dst, (reinterpret_cast<uintptr_t>(dst) & 15u) == 0, v, bytes, q[r]);
      }
    }
  }
  op_end(c);
}
