/*
 * b200ddp.h — C ABI of libb200ddp.so, the H100-native data plane behind the
 * `local_cuda` TorchX scheduler.
 *
 * This is the drop-in boundary for the data-parallel hot path.  The reference
 * (meta-pytorch/torchx) has no native code: its `dist.ddp` component only builds a
 * `torchrun` command line (torchx/components/dist.py:261-308) and the gradient
 * allreduce is executed by third-party torch + NCCL.  The entry points below are
 * therefore exactly the operations the reference's workers reach through
 * `torch.distributed` on this path, each citing the interface it replaces:
 *
 *   b2_comm_create     <- dist.init_process_group("nccl")   torchx/distributed/__init__.py:217-222
 *                         (TCPStore rendezvous + ncclCommInitRank; here: POSIX-shm control block +
 *                          CUDA-IPC exchange of one symmetric arena per rank over NVSwitch)
 *   b2_allreduce       <- the DDP bucket comm hook          torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py:18-93
 *                         (`buf.to(bf16).div_(W)` -> ncclAllReduce(SUM) -> `buf.copy_()`, 4 launches; here ONE fused kernel)
 *   b2_allreduce_op    <- `dist.all_reduce` of a metric      torchx/schedulers/test/train.py:35,
 *                                                           torchx/examples/apps/compute_world_size/module/util.py:37
 *                         (both SUM an int64 one-hot tensor)
 *   b2_allgather       <- `dist.all_gather_into_tensor` / `dist.all_gather`
 *   b2_reduce_scatter  <- `dist.reduce_scatter_tensor` / `dist.reduce_scatter`
 *   b2_reduce          <- `dist.reduce`
 *   b2_alltoall, b2_alltoall_max_bytes <- `dist.all_to_all_single` / `dist.all_to_all`
 *   b2_p2p             <- dist.send / dist.recv / dist.batch_isend_irecv (and the gather / scatter built on them)
 *   b2_batchnorm_stats <- torch's SyncBatchNorm forward: all_gather of (mean, invstd, count) + the count mask +
 *                         batch_norm_gather_stats_with_counts (torch/nn/modules/_functions.py)
 *   b2_allreduce_gather <- the Reducer's bucket copy-in fused into the hook (reducer.cpp mark_variable_ready_dense)
 *   b2_broadcast       <- DDP init / per-forward buffer sync torch/nn/parallel/distributed.py:881-890, 2176-2243
 *   b2_barrier         <- dist.barrier()                     torchx/distributed/__init__.py:268,274,297,303
 *   b2_comm_destroy    <- dist.destroy_process_group()
 *
 * Conventions: plain pointers and sizes only (no torch types); every function returns
 * B2_OK (0) or a negative B2_E* code and never throws across the ABI; the text of the
 * last error on the calling thread is available from b2_last_error().  All device work
 * is enqueued asynchronously on the caller's CUDA stream (`stream` is a cudaStream_t
 * passed as void*; NULL = the legacy default stream).  A communicator is a single
 * stream-ordered sequence of collectives (like an NCCL communicator): all ranks must
 * issue the same collectives in the same order, and calls on one communicator must not
 * be issued concurrently from several host threads.  Point-to-point calls (b2_p2p) involve
 * only the ranks they name; those of one communicator must be issued on one stream, or on
 * streams ordered against each other, because its channel counters are per-communicator state.
 */
#ifndef B200DDP_H_
#define B200DDP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_ABI_VERSION 3 /* 3: fp16 modes B2_F32_WIRE_F16 and B2_F16; later b2_allreduce_op, b2_allgather, b2_batchnorm_stats,
                            b2_reduce_scatter, b2_bn_*_elemt, b2_alltoall*, b2_reduce_scatter_step, b2_bn_reduce_plan, b2_bn_stats,
                            b2_bn_backward_reduce, b2_reduce and b2_reduce_scatter_step_bf16, which only add symbols: a binding that needs them
                            fails to resolve them against an older library */
#define B2_MAX_WORLD 8 /* one NVSwitch domain: 8 x H100 */

/* ---- return codes ---------------------------------------------------------------- */
#define B2_OK 0
#define B2_EINVAL (-1)   /* bad argument (null pointer, rank >= world, unknown dtype ...) */
#define B2_ECUDA (-2)    /* a CUDA runtime call failed; see b2_last_error() */
#define B2_ESYS (-3)     /* shm_open/mmap/... failed */
#define B2_ETIMEOUT (-4) /* rendezvous or an in-kernel peer wait timed out */
#define B2_ENOPEER (-5)  /* two ranks' devices cannot reach each other over P2P */
#define B2_ESTATE (-6)   /* communicator is poisoned by an earlier failure */
#define B2_ENOTSUP (-7)  /* the requested algorithm needs a capability this communicator lacks (b2_comm_caps) */

/* ---- element / wire formats ------------------------------------------------------ */
/* The arithmetic of every mode is fixed so results are bit-reproducible run to run and
 * independent of timing:   c_r = wire(scale * x_r) ;  s = ((c_0 + c_1) + ...) + c_{W-1} in fp32,
 * rank order ;  out = round(s).  See oracle/allreduce_oracle.c for the exact rounding points. */
#define B2_F32_WIRE_BF16 0 /* fp32 bucket, bf16 on the wire, fp32 result holding bf16-representable values
                              (== torch bf16_compress_hook semantics)                                   */
#define B2_F32 1           /* fp32 bucket, fp32 on the wire (== DDP default: pre-divide then SUM)         */
#define B2_BF16 2          /* bf16 bucket, bf16 on the wire, fp32 accumulate, one final rounding          */
#define B2_F32_WIRE_F16 3  /* fp32 bucket, fp16 on the wire, fp32 result holding fp16-representable values
                              (== torch fp16_compress_hook semantics):
                              c_r = f16(float(f16(x)) * scale),  out = float(f16(s))                      */
#define B2_F16 4           /* fp16 bucket, fp16 on the wire, fp32 accumulate, one final rounding
                              (== allreduce_hook / the hook-less Reducer on an fp16 bucket):
                              c_r = f16(float(x) * scale),  out = f16(s)                                  */
/* fp16 roundings are IEEE binary16 round-to-nearest-even: subnormals are kept, overflow goes to +-inf (never saturates:
 * GradScaler relies on an overflowed gradient arriving as inf on every rank), a NaN stays a NaN.  Mode numbers 5..7 are
 * unused and rejected. */

/* ---- algorithm selection --------------------------------------------------------- */
#define B2_ALGO_AUTO 0
#define B2_ALGO_ONESHOT 1      /* push whole message to every peer, one flag barrier, reduce locally                  */
#define B2_ALGO_TWOSHOT 2      /* push-scatter (fused cast) -> reduce own slice -> pull-gather (fused cast), one pass */
#define B2_ALGO_TWOSHOT_PIPE 3 /* the same three phases as warp-specialised roles pipelined over K chunks             */
#define B2_ALGO_NVLS 4         /* cast -> multimem.ld_reduce + multimem.st through the NVSwitch -> widen, pipelined;
                                  needs B2_CAP_MULTICAST.  The switch sums the W contributions with fp32 accumulation
                                  and rounds once; its summation order is the switch's, see DESIGN.md 2.4              */
#define B2_ALGO_TWOSHOT_LL 5   /* barrier-free two-shot: push-scatter -> reduce as contributions arrive -> push the result
                                  to every rank -> widen as slices arrive; arrival is read off the data itself (sentinel-
                                  filled buffers), no flag barrier and no fence on the data path; rank-order arithmetic   */

/* ---- capabilities (b2_comm_caps) -------------------------------------------------- */
#define B2_CAP_VMM 1       /* arena is a CUDA VMM allocation shared by file descriptor (else cudaMalloc + CUDA IPC) */
#define B2_CAP_MULTICAST 2 /* arena is bound into an NVSwitch multicast object on every rank: NVLS is available    */

typedef struct b2_comm b2_comm_t; /* opaque */

/* Library / ABI version (B2_ABI_VERSION this header was written for). */
int b2_version(void);

/* Text of the last error raised on the calling thread ("" if none). Never NULL. */
const char* b2_last_error(void);

/*
 * Create this rank's communicator.  All `world` ranks (one process per GPU) call this with the
 * same `shm_name` (a POSIX shm object name such as "/b2_<app_id>", handed out by the launcher
 * through the B2_SHM_NAME environment variable) and the same `epoch` (the launcher's restart
 * counter: a re-launched gang uses a new epoch so survivors never map a dead peer's memory).
 * `device` is the CUDA ordinal this rank is pinned to.  `stage_bytes` is the per-rank size of ONE
 * of the two symmetric staging buffers (0 = default 512 MiB); messages larger than what fits are
 * chunked internally.  `timeout_ms` bounds the rendezvous (0 = default 120 s).  The collectives of a
 * communicator are issued by all ranks in the same order; its point-to-point calls (b2_p2p) on one stream,
 * or on streams ordered against each other.
 */
int b2_comm_create(b2_comm_t** out, int rank, int world, int device, const char* shm_name,
                   uint64_t epoch, size_t stage_bytes, int timeout_ms);

/*
 * Create `world` communicators inside ONE process (out[0..world-1]), rank i on devices[i].
 * Devices may repeat (all ranks on one GPU): this is the single-GPU parity-test topology.  With
 * distinct devices it uses cudaDeviceEnablePeerAccess instead of CUDA IPC.
 */
int b2_comm_create_local(b2_comm_t** out, int world, const int* devices, size_t stage_bytes);

int b2_comm_destroy(b2_comm_t* comm);

int b2_comm_rank(const b2_comm_t* comm);
int b2_comm_world(const b2_comm_t* comm);
int b2_comm_device(const b2_comm_t* comm);

/* Bitmask of B2_CAP_* this communicator ended up with (identical on every rank), or B2_EINVAL. */
int b2_comm_caps(const b2_comm_t* comm);

/* In-kernel peer-wait timeout (default 600 s, NCCL's default for the same situation; B2_TIMEOUT_MS env overrides at
 * create time).  A kernel that gives up records B2_ETIMEOUT for b2_comm_status() and poisons the communicator. */
int b2_comm_set_timeout_ms(b2_comm_t* comm, int timeout_ms);

/* Upper bound on CTAs one collective may occupy (default: tuned per message size; 0 restores it).
 * Must be set identically on every rank. */
int b2_comm_set_max_ctas(b2_comm_t* comm, int max_ctas);

/*
 * What B2_ALGO_AUTO resolves to for a message of `n_elems` elements in `mode` on `world` ranks with the library's default
 * thresholds (and the B2_* environment overrides); `has_multicast` = the communicator would have B2_CAP_MULTICAST.  Pure
 * function, no GPU needed: lets a caller (and the CPU test-suite) see the policy table of DESIGN.md 2.6.  Messages larger
 * than a staging buffer are cut into several launches, each resolved on its own size.  world == 1: B2_ALGO_AUTO (local pass).
 */
int b2_auto_algo(int world, int mode, size_t n_elems, int has_multicast);

/*
 * Tuning knobs of the AUTO algorithm choice and of the pipelined kernels; must be set identically on every rank.
 *   "oneshot_max_bytes"  one-shot up to this many wire bytes           (env B2_ONESHOT_MAX_BYTES)
 *   "pipe_min_bytes"     pipelined two-shot from this many wire bytes   (env B2_PIPE_MIN_BYTES)
 *   "nvls_min_bytes"     NVLS from this many wire bytes                 (env B2_NVLS_MIN_BYTES)
 *   "nvls_min_world"     NVLS from this world size                      (env B2_NVLS_MIN_WORLD)
 *   "ll_min_bytes"       barrier-free LL two-shot from this many wire bytes (env B2_LL_MIN_BYTES) ...
 *   "ll_max_bytes"       ... up to (excluding) this many                (env B2_LL_MAX_BYTES)
 *   "pipe_chunk_bytes"   target wire bytes per pipeline chunk           (env B2_PIPE_CHUNK_KB, in KiB)
 *   "max_ctas"           same as b2_comm_set_max_ctas
 * And one test and diagnostic knob:
 *   "op_count"           sets the device op counter (see b2_comm_op_count) to `value`, so that a test can run collectives
 *                        where a long-lived communicator's counter would be.  Only while the communicator is idle, with
 *                        the same value on every rank; synchronises the device, then copies the value.
 */
int b2_comm_set_param(b2_comm_t* comm, const char* name, long long value);

/* The device op counter: the number of collectives this communicator has completed, plus any "op_count" it was given.
 * Point-to-point does not count.  A synchronous copy; 0 with b2_last_error() set if `comm` is NULL or the copy fails. */
uint64_t b2_comm_op_count(const b2_comm_t* comm);

/*
 * Non-blocking health check: B2_OK, B2_ETIMEOUT if any kernel of this communicator gave up
 * waiting for a peer (its output is then undefined), or B2_EINVAL if an all-to-all's split sizes
 * disagreed across ranks or exceeded the per-pair limit (see b2_alltoall), or a point-to-point
 * receive's byte count disagreed with its sender's (see b2_p2p).  Reads a host-mapped
 * status word; does not synchronise the device.  Either code poisons the communicator: every later
 * collective returns B2_ESTATE.
 */
int b2_comm_status(const b2_comm_t* comm);

/* Number of kernels this communicator has launched so far (for bench.py's gpu_launches). */
uint64_t b2_comm_launch_count(const b2_comm_t* comm);

/* B2_ALGO_* of the most recent multi-rank allreduce launch of this communicator (what B2_ALGO_AUTO resolved to; 0 if none). */
int b2_comm_last_algo(const b2_comm_t* comm);

/*
 * Measurement aid (tools/sweep_allreduce.py --trace): when enabled, every CTA of a collective records %globaltimer at
 * its phase boundaries, 8 u64 slots per CTA.  Single-pass kernels: start, scatter/push done, barrier 1 passed, reduce
 * done, barrier 2 passed, gather done.  Pipelined kernels (one stamp per role group): role A start, role A done (all
 * chunks), role B passed its first wait, role B done, role C passed its first wait, role C done.  Calling with a
 * non-NULL `out` first copies the stamps of the most recent collective for CTAs [0, max_ctas) (synchronously; call
 * after a stream sync), then applies `enable`.
 */
int b2_comm_trace(b2_comm_t* comm, int enable, uint64_t* out, int max_ctas);

/*
 * In-place averaged/scaled SUM allreduce of `n_elems` elements at device pointer `buf`
 * (any device allocation of this rank; it does not need to be symmetric memory):
 *      buf[i] <- round( sum_{r=0..W-1} wire( scale * buf_r[i] ) )
 * `mode` is one of B2_F32_WIRE_BF16 / B2_F32 / B2_BF16 / B2_F32_WIRE_F16 / B2_F16, `algo` one of B2_ALGO_*.
 * scale is normally 1/W (DDP gradient averaging).  n_elems == 0 is a no-op.
 */
int b2_allreduce(b2_comm_t* comm, void* buf, size_t n_elems, int mode, float scale, int algo,
                 void* stream);

/*
 * The same collective with the INPUT gathered straight from the per-parameter gradient tensors instead of from the
 * bucket: replaces the Reducer's copy-in pass (torch/csrc/distributed/c10d/reducer.cpp, mark_variable_ready_dense ->
 * bucket_view.copy_(grad); with gradient_as_bucket_view the copy still happens whenever autograd produced the gradient
 * elsewhere, torch/nn/parallel/distributed.py:589-600) - 8 bytes per element and one multi-tensor launch per bucket.
 *      out[i] <- round( sum_r wire( scale * segment_r(i)[i - begin] ) ),   i in [0, n_elems)
 * `segments`: HOST array of 1..B2_MAX_SEGMENTS entries in bucket order and without gaps: segment k covers bucket elements
 * [begin, end) and reads them from the DEVICE pointer `src` (this rank's tensor of the bucket's dtype, dense in the
 * bucket's element order; it may alias `out`).  The table is copied into the kernel parameters by this call: it need not
 * outlive it.  `out` is this rank's bucket.  More parameters than B2_MAX_SEGMENTS: B2_EINVAL (copy in, then b2_allreduce).
 * A segment whose `src` is B2_SEGMENT_ZEROS contributes +0.0 for each of its elements, exactly as a zero-filled tensor of
 * the bucket's dtype would, and is not read from memory (a parameter that got no gradient in this step).  A NULL `src`
 * is B2_EINVAL.
 */
#define B2_MAX_SEGMENTS 128
/* The `src` of a zero segment: not NULL, and misaligned for every element type, so no tensor has it. */
#define B2_SEGMENT_ZEROS ((const void*)1)
typedef struct b2_segment {
  const void* src;
  uint64_t begin;
  uint64_t end;
} b2_segment_t;

int b2_allreduce_gather(b2_comm_t* comm, void* out, size_t n_elems, const b2_segment_t* segments, int n_segments,
                        int mode, float scale, int algo, void* stream);

/* Broadcast `bytes` bytes at `buf` from rank `root` to every rank (bit-exact copy). */
int b2_broadcast(b2_comm_t* comm, void* buf, size_t bytes, int root, void* stream);

/*
 * Exact collectives (DESIGN.md 2.4).  `dtype` is a B2_DT_*, `op` a B2_OP_*:
 *   int32, int64                 SUM wraps (two's complement, modulo 2^32 / 2^64); MIN / MAX exact.
 *   float32, bfloat16, float16   MIN / MAX exact: a NaN at any rank gives a NaN (its payload is unspecified but the same on
 *                                every rank), otherwise IEEE 754-2019 minimum / maximum with -0.0 < +0.0; +-inf are
 *                                ordinary values.
 *                                SUM / AVG run b2_allreduce in B2_F32 / B2_BF16 / B2_F16 with scale 1 / (1/W) and
 *                                B2_ALGO_AUTO: the rank-order fp32 sum with one final rounding (equal to NCCL at W = 2 only).
 * The integer and MIN / MAX results are the same bits on every rank and do not depend on timing.  AVG on an integer
 * dtype, any other op (PRODUCT, bitwise ...) and any other dtype are B2_EINVAL.
 */
#define B2_DT_INT32 0
#define B2_DT_INT64 1
#define B2_DT_FLOAT32 2
#define B2_DT_BFLOAT16 3
#define B2_DT_FLOAT16 4
#define B2_OP_SUM 0
#define B2_OP_AVG 1
#define B2_OP_MIN 2
#define B2_OP_MAX 3

/* In place: buf[i] <- op_r buf_r[i] over `n_elems` elements (contract above).  n_elems == 0 is a no-op; W == 1 leaves
 * `buf` as it is. */
int b2_allreduce_op(b2_comm_t* comm, void* buf, size_t n_elems, int dtype, int op, void* stream);

/* out[r*bytes .. (r+1)*bytes) <- rank r's `in` (bit-exact copy).  `in` may be exactly this rank's block of `out` (torch's
 * in-place form); any other overlap of `in` and `out` is B2_EINVAL.  bytes == 0 is a no-op. */
int b2_allgather(b2_comm_t* comm, void* out, const void* in, size_t bytes, void* stream);

/* out[i] <- op_r in_r[rank*n_elems + i], i < n_elems; `in` holds W*n_elems elements (block r for rank r).  Same dtypes,
 * ops and arithmetic contract as b2_allreduce_op: rank r's `out` is block r of what b2_allreduce_op of the same inputs
 * leaves on every rank, bit for bit, except where that allreduce's B2_ALGO_AUTO picked B2_ALGO_NVLS (the reduce-scatter
 * always sums in rank order).  `out` may be exactly this rank's block of `in` (the in-place form); any other overlap is
 * B2_EINVAL.  n_elems == 0 is a no-op; at W == 1 it copies the block (nothing if in place).  Each rank sends and
 * receives (W-1)/W of its input. */
int b2_reduce_scatter(b2_comm_t* comm, void* out, const void* in, size_t n_elems, int dtype, int op, void* stream);

/* In place on the root: buf[i] <- op_r buf_r[i] over `n_elems` elements on rank `root`; every other rank's `buf` is only
 * read.  Same dtypes, ops and arithmetic contract as b2_allreduce_op: the root's `buf` is what b2_allreduce_op of the same
 * inputs leaves, bit for bit, except where that allreduce's B2_ALGO_AUTO picked B2_ALGO_NVLS, and it is the concatenation
 * of the W blocks b2_reduce_scatter leaves.  Checked in b2_allreduce_op's order: dtype and op (even when n_elems == 0),
 * then n_elems == 0 is a no-op, then a null communicator or buffer, a root outside [0, W) (B2_EINVAL) and a poisoned
 * communicator (B2_ESTATE).  W == 1 leaves `buf` as it is.  Each rank sends (W-1)/W of its input; the root also receives
 * (W-1)/W of it. */
int b2_reduce(b2_comm_t* comm, void* buf, size_t n_elems, int dtype, int op, int root, void* stream);

/*
 * The gradient reduce-scatter of a sharded bucket (the mini-DDP's ZeRO-1 mode), with its input gathered from a segment
 * table as in b2_allreduce_gather:
 *      out[i] <- round( sum_r wire( scale * segment_r(rank*block + i) ) ),   i in [0, block)
 * The table covers the padded bucket [0, W*block) in bucket order without gaps, with the rules and error texts of
 * b2_allreduce_gather, B2_SEGMENT_ZEROS included; `mode` is any of the five B2_* gradient modes.  out[0, block) is this rank's block of what
 * b2_allreduce_gather of the same table leaves, bit for bit, wherever that allreduce runs a rank-order kernel (every
 * algorithm but B2_ALGO_NVLS).  An unknown mode is B2_EINVAL; block == 0 is a no-op; a poisoned communicator is
 * B2_ESTATE.  At W == 1 the call is the local pass of b2_allreduce_gather, with its rounding.  Each rank sends and
 * receives (W-1)/W of the wire data.
 */
int b2_reduce_scatter_gather(b2_comm_t* comm, void* out, size_t block, const b2_segment_t* segments, int n_segments, int mode,
                             float scale, void* stream);

/*
 * The same reduce-scatter with the optimizer step fused into it (the ZeRO-1 mini-DDP's overlap_with_ddp mode): instead of
 * storing this rank's reduced block, the kernel steps this rank's block of the flat fp32 parameter buffer and its optimizer
 * state with it, element by element, with the arithmetic of torch's fused optimizers (torch._fused_sgd_, _fused_adam_,
 * _fused_adamw_; fp32 parameters, no grad scale, no amsgrad):
 *      g[i] = round( sum_r wire( scale * segment_r(rank*block + i) ) )   (what b2_reduce_scatter_gather stores)
 *      param[i], state[i] <- step(group of i, param[i], g[i], state[i]),  i in [0, block)
 * The segment table takes B2_SEGMENT_ZEROS segments as b2_reduce_scatter_gather's does.
 * `opt->param`, `opt->state0` and `opt->state1` point at `block` fp32 elements each: this rank's block of the parameter
 * buffer, then momentum_buffer (SGD) or exp_avg and exp_avg_sq (Adam / AdamW).  The runs of `opt` assign block elements to
 * parameter groups: run k covers block elements [run_begin[k], run_begin[k+1]) (run_begin[0] == 0, increasing,
 * run_begin[n_runs] == block), and an element of a run whose group is B2_OPT_NO_GROUP (the pad) is not touched.
 * Modes B2_F32_WIRE_BF16, B2_F32 and B2_F32_WIRE_F16 only.  B2_EINVAL, before anything is launched, for: the checks of
 * b2_reduce_scatter_gather, another mode, an unknown kind, a null `opt` or parameter pointer, a null state pointer the kind
 * reads, 0 or more than B2_OPT_MAX_GROUPS groups, 0 or more than B2_OPT_MAX_RUNS runs, runs that do not tile the block, a
 * group index out of range, or block >= 2^32.
 */
#define B2_OPT_SGD 1
#define B2_OPT_ADAM 2
#define B2_OPT_ADAMW 3
#define B2_OPT_MAX_GROUPS 8
#define B2_OPT_MAX_RUNS 128
#define B2_OPT_NO_GROUP 255
typedef struct b2_optim_group {
  double lr;
  double weight_decay;
  double momentum;  /* SGD */
  double dampening; /* SGD */
  double beta1;     /* Adam / AdamW */
  double beta2;     /* Adam / AdamW */
  double eps;       /* Adam / AdamW */
  int nesterov;     /* SGD */
  int maximize;
} b2_optim_group_t;

typedef struct b2_optim {
  int kind;     /* B2_OPT_* */
  int n_groups; /* 1..B2_OPT_MAX_GROUPS */
  int n_runs;   /* 1..B2_OPT_MAX_RUNS */
  float* param;
  float* state0; /* SGD: momentum_buffer (may be NULL when every group's momentum is 0); Adam / AdamW: exp_avg */
  float* state1; /* Adam / AdamW: exp_avg_sq; SGD: unused */
  uint64_t run_begin[B2_OPT_MAX_RUNS + 1];
  uint8_t run_group[B2_OPT_MAX_RUNS];
  float run_step[B2_OPT_MAX_RUNS]; /* Adam / AdamW: the step count of this update (>= 1); SGD: 1 on the first step, else 0 */
  /* Adam only (its rounding of param * weight_decay depends on where an element sits in its parameter tensor, see
   * DESIGN.md 2.4): the index within its parameter of the run's first element, and 1 if torch's fused Adam steps that
   * parameter on its scalar path (numel not a multiple of 4, or not 16-byte aligned), else 0.  A run then lies within one
   * parameter.  Ignored by the other kinds. */
  uint64_t run_index[B2_OPT_MAX_RUNS];
  uint8_t run_scalar[B2_OPT_MAX_RUNS];
  b2_optim_group_t group[B2_OPT_MAX_GROUPS];
} b2_optim_t;

int b2_reduce_scatter_step(b2_comm_t* comm, size_t block, const b2_segment_t* segments, int n_segments, int mode, float scale,
                           const b2_optim_t* opt, void* stream);

/*
 * The same fused step for a bf16 bucket whose parameters have fp32 master weights (the ZeRO-1 mini-DDP's
 * master_weights=True with overlap_with_ddp): mode B2_BF16, and the step updates this rank's block of the masters, not
 * of the bf16 parameters, which it then writes from them:
 *      g[i] = float( round_bf16( sum_r bf16( scale * segment_r(rank*block + i) ) ) )   (b2_reduce_scatter_gather's bits, widened)
 *      master[i], state[i] <- step(group of i, master[i], g[i], state[i])
 *      param_bf16[i] <- bf16(master[i])   (round to nearest even, NaN -> 0x7FFF: ATen's conversion on the device)
 * for every element i of a run with a group; pad elements are not touched.  `opt->param` points at this rank's `block`
 * fp32 masters, `param_bf16` at this rank's block of the bucket's bf16 parameter buffer; the state and runs are those of
 * b2_reduce_scatter_step.  B2_EINVAL, before anything is launched, for the checks of b2_reduce_scatter_step (the mode
 * check aside) and a null or not 16-byte aligned `param_bf16`.  At W == 1 the gradient is the local pass's rounding, as for fp32 buckets.
 */
int b2_reduce_scatter_step_bf16(b2_comm_t* comm, size_t block, const b2_segment_t* segments, int n_segments, float scale,
                                const b2_optim_t* opt, void* param_bf16, void* stream);

/*
 * All-to-all, a bit-exact copy of bytes (any dtype): out[r] <- the recv_bytes[r] bytes rank r sends this rank, in[j] is what
 * goes to rank j (send_bytes[j] bytes).  The four arrays are HOST arrays of W entries indexed by rank, copied into the kernel
 * parameters by the call; a pointer whose count is 0 may be NULL.  No `out` range may overlap another `out` range or any
 * `in` range (there is no in-place form).  One launch per call whatever the sizes, so each (sender, receiver) pair of
 * distinct ranks carries at most b2_alltoall_max_bytes(comm) bytes (a rank's block to itself is copied directly and has
 * no limit).  Each rank sends and receives (W-1)/W of its data when the splits are even.
 *   - A null communicator or array, a null pointer with a non-zero count, or an overlap: B2_EINVAL before anything is
 *     launched; a poisoned communicator: B2_ESTATE.
 *   - A pair over the limit: its sender's and its receiver's calls return B2_EINVAL, but still launch so that no rank
 *     waits for them; every rank's kernel then gives up the exchange, writes no output and records B2_EINVAL for
 *     b2_comm_status, which poisons every rank's communicator.
 *   - recv_bytes[r] different from what rank r sends this rank (send_bytes[rank] vs recv_bytes[rank] included): only this
 *     rank's kernel sees it.  It writes none of this rank's outputs and records B2_EINVAL, poisoning this rank's
 *     communicator; the other ranks complete normally.  At W == 1 the call returns B2_EINVAL instead.
 * At W > 1 a rank whose counts are all 0 still takes part (the other ranks' barriers include it).  At W == 1 the call is
 * one device-to-device copy.
 */
int b2_alltoall(b2_comm_t* comm, void* const* out, const size_t* recv_bytes, const void* const* in, const size_t* send_bytes,
                void* stream);

/* The most bytes one rank may send another in one b2_alltoall: a stage region less its 16-byte count header (the stage
 * size is b2_comm_create's stage_bytes, default 512 MiB, divided into W + 1 regions).  0 for a null communicator. */
size_t b2_alltoall_max_bytes(const b2_comm_t* comm);

/*
 * Point-to-point: a batch of 1..B2_P2P_MAX_OPS sends and receives, a bit-exact copy of bytes (any dtype), in ONE launch.
 * `ops` is a HOST array copied into the kernel parameters by the call.  A send gives `bytes` bytes at `ptr` to rank
 * `peer`; a receive writes into `ptr` the next message rank `peer` sends this rank, which must have exactly `bytes` bytes.
 * Messages between an ordered pair of ranks (a channel) match in issue order, as NCCL's do; a batch may hold several ops
 * on one channel (they run in list order) and ops on any other channels, and it never waits on itself: ops of one batch
 * make progress whatever their order in the list and in the peer's batch.  send / recv / isend / irecv are batches of one.
 *   - A null communicator or op list, n_ops outside 1..B2_P2P_MAX_OPS, a peer out of range or equal to this rank (which
 *     rules out W == 1), a null pointer with a non-zero byte count, or a receive range that overlaps any other range of the
 *     batch: B2_EINVAL before anything is launched; a poisoned communicator: B2_ESTATE.
 *   - Every wait is bounded: a kernel that gives up records B2_ETIMEOUT for b2_comm_status.  Once a wait of this
 *     communicator has given up, or a receive has found a size mismatch, its other waits give up within a few polls
 *     instead of a timeout each.  A chunk whose wait gave up is neither written nor handed on, so a receiver that arrives
 *     after its sender gave up waits for it and records its own timeout rather than taking stale bytes.
 *   - A receive whose byte count is not the sender's: the receiver writes none of that message and records B2_EINVAL,
 *     which poisons only its own communicator.  A sender whose message is at most b2_p2p_eager_bytes has already
 *     finished; a larger one waits for the slots the receiver never hands back until its timeout.  A receiver that
 *     expects more chunks than its sender sent stops waiting for the missing ones once it has recorded the mismatch.
 *   - Deadlocks the caller can create: two ranks that each send more than b2_p2p_eager_bytes before their recv, in
 *     separate calls, wait until the timeout, exactly as with NCCL outside a group; the cure is one batch.  The same holds
 *     for a point-to-point call ordered on one rank against a collective that the peer issues in the opposite order.
 * Point-to-point uses its own buffers and counters and never touches the collectives' state, so a collective's result and
 * protocol are the same whatever point-to-point traffic runs before, after or between collectives.
 */
#define B2_P2P_MAX_OPS 64
typedef struct b2_p2p_op {
  int peer;    /* the other rank */
  int is_send; /* nonzero: send, 0: receive */
  void* ptr;   /* device pointer of this rank (may be NULL when bytes == 0) */
  size_t bytes;
} b2_p2p_op_t;

int b2_p2p(b2_comm_t* comm, const b2_p2p_op_t* ops, int n_ops, void* stream);

/* The largest message a send completes without the matching receive having been launched, once the earlier messages on
 * its channel have been received: the inbox of K slots of one chunk each, less their 16-byte headers (8 x 512 KiB - 128
 * bytes).  0 for a null communicator. */
size_t b2_p2p_eager_bytes(const b2_comm_t* comm);

/*
 * SyncBatchNorm statistics: in place, mean[c] / invstd[c] <- the merge of every rank's (mean, invstd, count) over the ranks
 * with count >= 1, in rank order, with the arithmetic of ATen's batch_norm_gather_stats_with_counts (DESIGN.md 2.4);
 * running_mean / running_var (fp32, either may be NULL) updated in place; counts_out (W floats, may be NULL) <- every
 * rank's count in rank order.  channels == 0 is a no-op.
 * Replaces the statistics exchange of torch's SyncBatchNorm forward (torch/nn/modules/_functions.py: torch.cat of
 * mean / invstd / count -> dist.all_gather_into_tensor -> the count >= 1 mask, a device-to-host sync -> counts.to() ->
 * torch.batch_norm_gather_stats_with_counts) with one kernel and no host sync.  mean, invstd and the row's count must
 * fit one stage region (B2_EINVAL otherwise); a negative or NaN count is B2_EINVAL.  At W == 1 the merge runs on this
 * rank's row alone.
 */
int b2_batchnorm_stats(b2_comm_t* comm, float* mean, float* invstd, float count, size_t channels,
                       float* running_mean, float* running_var, double momentum, double eps,
                       float* counts_out, void* stream);

/*
 * The elementwise passes of training-mode BatchNorm2d on channels-last activations (no communicator; DESIGN.md 2.3 / 2.4).
 * The data is the row-major [rows, channels] view of an NHWC-contiguous tensor (rows = N*H*W); x, y, dy and dx are `dtype`
 * (B2_DT_BFLOAT16, the one format whose torch BatchNorm runs ATen's own kernels rather than cuDNN's), 16-byte aligned; every
 * other array is float32 [channels].  The reductions are ATen's
 * (torch.batch_norm_update_stats, torch.batch_norm_backward_reduce) and the arithmetic here is ATen's, expression for
 * expression, so the results are the bits ATen's own BatchNorm computes.  eps is converted to float as ATen's launch does.
 * No call allocates or synchronises the host.  channels % 8 != 0, rows < 2, an unknown dtype, a null or a misaligned
 * pointer is B2_EINVAL.
 */
/* save_invstd <- rsqrt(var + eps) (var: the biased batch variance); y <- weight * (x - mean) * save_invstd + bias. */
int b2_bn_forward_elemt(const void* x, void* y, size_t rows, size_t channels, int dtype, const float* weight, const float* bias,
                        const float* mean, const float* var, double eps, float* save_invstd, int device, void* stream);

/* dx <- (dy - sum_dy / rows - (x - mean) * invstd^2 * sum_dy_xmu / rows) * invstd * weight. */
int b2_bn_backward_elemt(const void* dy, const void* x, void* dx, size_t rows, size_t channels, int dtype, const float* weight,
                         const float* mean, const float* invstd, const float* sum_dy, const float* sum_dy_xmu, int device,
                         void* stream);

/*
 * The two reductions of training-mode BatchNorm2d on the same [rows, channels] view, with the bits of ATen's channels-last
 * kernels (batch_norm_collect_statistics_channels_last_kernel and the running-statistics update of batch_norm_update_stats;
 * batch_norm_backward_reduce_channels_last_kernel): the same reduction tree, order and contractions (DESIGN.md 2.4).  They
 * cover the inputs ATen reduces with those kernels: rows * channels < 2^31 - 1 (B2_EINVAL above), plus the checks of the
 * elementwise passes.  A layer whose tree has more than one CTA row (geometry[3] > 1) needs a float-aligned device
 * workspace of the size b2_bn_reduce_plan reports (0 otherwise, and then workspace may be null); it is scratch, ordered
 * on `stream`, and a second small kernel folds it.  No call allocates, synchronises the host or uses atomics.
 */
/* ATen's launch geometry for the layer, geometry = {block.x, block.y, grid.x, grid.y}, and the workspace size in bytes. */
int b2_bn_reduce_plan(size_t rows, size_t channels, int* geometry, size_t* workspace_bytes);

/* mean, var <- the batch mean and biased variance (m2n / rows); if running_mean / running_var are given (both or neither):
 * running <- (1 - momentum) * running + momentum * (mean, var * rows / (rows - 1)), momentum converted to float. */
int b2_bn_stats(const void* x, size_t rows, size_t channels, int dtype, float* mean, float* var, float* running_mean, float* running_var,
                double momentum, void* workspace, size_t workspace_bytes, int device, void* stream);

/* sum_dy <- sum(dy), sum_dy_xmu <- sum(dy * (x - mean)), grad_weight <- sum_dy_xmu * invstd, grad_bias <- sum_dy. */
int b2_bn_backward_reduce(const void* dy, const void* x, size_t rows, size_t channels, int dtype, const float* mean, const float* invstd,
                          float* sum_dy, float* sum_dy_xmu, float* grad_weight, float* grad_bias, void* workspace, size_t workspace_bytes,
                          int device, void* stream);

/* Device-side barrier across all ranks, ordered on `stream`. */
int b2_barrier(b2_comm_t* comm, void* stream);

/*
 * Local (no peers) building block, also the W==1 fast path of b2_allreduce: applies
 * x <- round(wire(scale*x)) to `n_elems` elements on `device`.  Exposed so the single-GPU
 * roofline of the fused cast/scale pass can be measured without a communicator.
 */
int b2_local_pass(void* buf, size_t n_elems, int mode, float scale, int device, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200DDP_H_ */
