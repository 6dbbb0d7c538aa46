/*
 * traceml_b200.h -- C-ABI of libtraceml_b200.so, the GPU-native telemetry engine (H100, sm_90a).
 *
 * The reference (traceopt-ai/traceml v0.2.15) is pure Python and has no FFI;
 * its "operator API" for this path is the set of Python seams listed in
 * SURVEY.md section 8(b).  Each entry point below names the seam it replaces
 * (paths relative to the reference's src/traceml/).  INTEGRATION.md shows the
 * ctypes stub a reference maintainer would add at each seam.
 *
 * Conventions
 *   - every function returns TML_OK (0) or a negative tml_status; none throws;
 *   - "stream" is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - functions in the STEP PATH group never synchronise the host with the
 *     device (no cudaStreamSynchronize / cudaDeviceSynchronize / blocking copy);
 *   - functions in the REDUCE group run at summary time, off the step path,
 *     and may synchronise the stream they are given;
 *   - plain pointers and sizes only: no torch / pybind types cross this ABI.
 */
#ifndef TRACEML_B200_H_
#define TRACEML_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TML_ABI_VERSION 1u

#define TML_N_PHASES 6u   /* canonical phases, renderers/step_time/compute.py:24-31 */
#define TML_MAX_PHASES 8u /* accumulator slots (6 canonical + "other" + spare)     */
#define TML_MAX_RANKS 64u

/* phase ids == WindowRow column order (SURVEY 8d) */
enum tml_phase {
  TML_PHASE_DATALOADER = 0, /* _traceml_internal:dataloader_next  (host clock) */
  TML_PHASE_H2D = 1,        /* _traceml_internal:h2d_time                       */
  TML_PHASE_FORWARD = 2,    /* _traceml_internal:forward_time                   */
  TML_PHASE_BACKWARD = 3,   /* _traceml_internal:backward_time                  */
  TML_PHASE_OPTIMIZER = 4,  /* _traceml_internal:optimizer_step                 */
  TML_PHASE_STEP = 5,       /* _traceml_internal:step_time        (host clock) */
  TML_PHASE_OTHER = 6       /* any other user region: timed, not summarised     */
};

typedef enum tml_status {
  TML_OK = 0,
  TML_ERR_CUDA = -1,        /* a CUDA runtime call failed: see tml_last_error() */
  TML_ERR_ARG = -2,         /* bad argument                                     */
  TML_ERR_STATE = -3,       /* call out of sequence / context not initialised   */
  TML_ERR_NOMEM = -4,
  TML_ERR_NONMONOTONIC = -5,/* step ids decrease inside the retained ring       */
  TML_ERR_UNSUPPORTED = -6,
  TML_ERR_CAPTURE = -7,     /* stream is being captured into a CUDA graph       */
  TML_ERR_SMALL = -8        /* output buffer too small                          */
} tml_status;

/* ------------------------------------------------------------------ records */

/* 128 B / step / rank.  Replaces StepTimeBatch(+TimeEvent list) and
 * StepMemoryEvent: utils/timing.py:44-105, utils/step_memory.py:17-27. */
typedef struct tml_step_record {
  uint64_t step;
  uint64_t dur_ns[TML_N_PHASES];  /* summed per phase within the step      */
  uint32_t n_calls[TML_N_PHASES]; /* occurrences summed (a7: n_calls)      */
  uint64_t peak_alloc;            /* max_memory_allocated, bytes           */
  uint64_t peak_resv;             /* max_memory_reserved, bytes            */
  double host_ts;                 /* unix seconds at commit (row ts)       */
  uint32_t gpu_mask;              /* bit p: phase p was device-timed       */
  uint32_t flags;                 /* TML_REC_* */
  uint64_t seq;                   /* 0-based commit index on this rank     */
  uint64_t _pad;
} tml_step_record;

#define TML_REC_HAS_MEM 1u /* peaks are real (model lives on a CUDA device) */

/* 64 B / step / rank, the reduce's working row (ms, bytes as f64). */
typedef struct tml_window_row {
  double dataloader, h2d, forward, backward, optimizer, step_wall;
  double peak_alloc, peak_resv;
} tml_window_row;

/* 64 B / sample / rank.  Replaces ProcessSample: samplers/schema/process.py:89-150. */
typedef struct tml_proc_record {
  uint64_t seq;
  double ts;
  double cpu_pct;
  uint64_t rss;
  uint64_t mem_alloc;
  uint64_t mem_resv;
  uint64_t mem_total;
  uint32_t flags; /* TML_PROC_* */
  uint32_t cpu_cores;
} tml_proc_record;

#define TML_PROC_GPU_AVAILABLE 1u
#define TML_PROC_HAS_GPU_METRICS 2u

/* Running per-phase statistics kept on the device by the commit kernel
 * (warp-shuffle scan over a 256-bin log histogram); feeds the live view. */
typedef struct tml_live_phase {
  uint64_t count;     /* steps in which the phase ran   */
  uint64_t sum_ns;
  uint64_t worst_ns;  /* running max                    */
  uint64_t median_ns; /* running median (bin centre, +-6 %) */
} tml_live_phase;

typedef struct tml_live_stats {
  uint64_t steps_committed;
  tml_live_phase phase[TML_MAX_PHASES];
} tml_live_stats;

typedef struct tml_ctx tml_ctx; /* one engine per (process, GPU) */

/* ---------------------------------------------------------------- lifecycle */

/* Replaces TraceMLRuntime.__init__/start (runtime/runtime.py:66-95,142-160):
 * allocates the HBM rings, the host-mapped drain mirror and the in-flight
 * accumulators on `device`.  ring_slots >= 1; the reference retains
 * 1.5 x window rows (reporting/config.py:13-35). */
int tml_init(int device, int rank, int world, uint32_t ring_slots,
             uint32_t proc_slots, tml_ctx** out);
/* Replaces TraceMLRuntime.stop (runtime/runtime.py:163-193). */
int tml_shutdown(tml_ctx* ctx);
uint32_t tml_abi_version(void);
const char* tml_last_error(void);
const char* tml_status_str(int status);

/* ---------------------------------------------------------------- STEP PATH
 * No host synchronisation in this group. */

/* Open a device-timed region on `stream`: launches the 1-warp stamp kernel
 * (reads %globaltimer).  Returns a slot id >= 0 to pass to tml_phase_end, or a
 * negative tml_status.  Replaces the start half of timed_region(use_gpu=True):
 * utils/timing.py:202-210 (get_cuda_event x2 + start_evt.record()). */
int tml_phase_begin(tml_ctx* ctx, uint32_t phase, void* stream);
/* Close it: stamp kernel accumulates (end - begin) ns and n_calls into the
 * in-flight record of the open step.  Replaces utils/timing.py:226-249
 * (end_evt.record() + TimeEvent + record_event). */
int tml_phase_end(tml_ctx* ctx, uint32_t phase, int slot, void* stream);
/* Host-clock region (use_gpu=False, or no device work): add dur_ns / one call.
 * Replaces timed_region(use_gpu=False): utils/timing.py:211-213,236-244. */
int tml_phase_host(tml_ctx* ctx, uint32_t phase, uint64_t dur_ns);
/* Close the step: commit kernel stages the in-flight record through shared
 * memory, merges the host-clock phases and the allocator peaks (c10 allocator
 * counters are host state: they travel as launch arguments), writes one
 * coalesced 128-B line into the HBM ring, updates the running statistics and
 * bumps the head.  It writes NOTHING to host memory and issues no system-scope
 * fence: the training stream pays for the record, not for the sampler.
 * Replaces StepMemoryTracker.record + flush_step_events:
 * utils/step_memory.py:60-110, utils/flush_buffers.py:24-33,
 * utils/timing.py:163-180. */
int tml_step_commit(tml_ctx* ctx, uint64_t step, uint64_t peak_alloc,
                    uint64_t peak_resv, uint32_t flags, double host_ts,
                    void* stream);
/* Drop whatever the open step accumulated (TRACEML_DISABLED / failed setup). */
int tml_step_discard(tml_ctx* ctx);

/* ------------------------------------------------------- SAMPLER-SIDE (host)
 * Called from the sampler thread; never touches the training stream. */

/* Drain of completed records.  The sampler fetches them itself: one small copy
 * kernel (k_mirror) on the context's own sampler stream brings the records
 * committed since the last call -- and the live statistics -- into a host-mapped
 * mirror; the call waits for that stream only, never for the training stream.
 * Replaces StepTimeSampler.sample + StepMemorySampler.sample:
 * samplers/step_time_sampler.py:104-128, samplers/step_memory_sampler.py:12-65. */
int tml_drain(tml_ctx* ctx, tml_step_record* out, uint32_t max_records,
              uint32_t* n_out, uint64_t* n_dropped);
int tml_live(tml_ctx* ctx, tml_live_stats* out);
/* One process sample -> 64-B record committed on `stream` (side stream).
 * Replaces ProcessSampler.sample: samplers/process_sampler.py:208-238. */
int tml_proc_commit(tml_ctx* ctx, const tml_proc_record* sample, void* stream);
int tml_proc_drain(tml_ctx* ctx, tml_proc_record* out, uint32_t max_records,
                   uint32_t* n_out, uint64_t* n_dropped);
uint64_t tml_step_count(tml_ctx* ctx); /* records committed so far */
uint64_t tml_launch_count(tml_ctx* ctx); /* kernels launched by this context */
uint64_t tml_proc_count(tml_ctx* ctx);

/* Bulk append of already-formed records from HOST memory (replay, resume,
 * or a rank that spooled to disk): one async H2D copy per contiguous span. */
int tml_ring_load(tml_ctx* ctx, const tml_step_record* host_records, uint64_t n,
                  void* stream);
int tml_proc_load(tml_ctx* ctx, const tml_proc_record* host_records, uint64_t n,
                  void* stream);
int tml_ring_reset(tml_ctx* ctx);

/* -------------------------------------------------------------------- REDUCE
 * Cross-rank window reduce, in stages so the host can put its collectives
 * (torch.distributed / NCCL) between them.  kind: 0 = step-time window (last W
 * rows), 1 = step-memory window (all retained rows as candidates).           */

#define TML_KIND_TIME 0u
#define TML_KIND_MEM 1u

typedef struct tml_win_info {
  uint64_t n_retained;   /* rows linearised from the ring                     */
  uint64_t latest_step;  /* MAX(step) over retained rows (training_steps - 1) */
  uint32_t monotone;     /* 1 if step ids never decrease                      */
  uint32_t dup_rows;     /* rows repeating the previous step id               */
  /* per kind: candidate rows and [lo, hi] of their step ids (valid if n > 0) */
  uint64_t n_rows[2];
  uint64_t n_cand[2];    /* rows that enter alignment (usable/deduped)        */
  uint64_t lo[2];
  uint64_t hi[2];
  /* unaligned per-rank Step-Time window sums over the last W rows
   * (reporting/sections/step_time/model.py:203-281): dl, fwd, bwd, opt,
   * step_cpu(raw), traced, total; and the row count n                        */
  double t_sums[7];
  uint64_t t_count;
  /* rows that are candidates of BOTH kinds: n_both == n_cand[0] == n_cand[1]
   * means the time and memory candidate sets are the same rows               */
  uint64_t n_both;
  /* per kind: 1 if every window row is a candidate and their step ids are
   * consecutive (then tml_win_select_dense applies)                          */
  uint32_t dense[2];
  double kernel_ms;      /* device time of k_window_rows alone (CUDA events)   */
} tml_win_info;

/* Stage 1 (local).  Linearises the ring into WindowRows (ns -> ms), step ids
 * and row flags; computes the bounds above.  Replaces the per-rank half of
 * load_step_time_section_data / build_rank_summary and the candidate query of
 * the step-memory loader: reporting/sections/step_time/loader.py:44-72,
 * step_time/model.py:162-281, step_memory/loader.py:112-205. */
/* Reference-order sums (K3e, csrc/tml_exact_sum.h) may run BESIDE the row exchange instead of in
 * front of it: with ``on`` != 0 tml_win_prepare launches them on the context's side stream and
 * returns the deterministic tree sums in tml_win_info.t_sums; tml_win_exact_collect then yields
 * the reference-order sums (model.py:262-268 order) once they are needed -- at the end of the
 * reduce, for the per-rank summaries and the rank tie-breaks.  Off by default (stage-by-stage
 * callers get exact sums directly).                                                       */
int tml_win_set_defer(tml_ctx* ctx, int on);

int tml_win_exact_collect(tml_ctx* ctx, void* stream, double t_sums[7]);
/* rows the last K3e walk had to add one by one, per chain (diagnostic) */
int tml_win_exact_stats(tml_ctx* ctx, uint64_t slow_rows[7]);

int tml_win_prepare(tml_ctx* ctx, uint32_t window, void* stream,
                    tml_win_info* out);

/* Stage 2 (local).  Presence bytes (0/1) of this rank over step ids
 * [glo, glo + span) into caller memory `presence_dev` (device, span bytes).
 * The caller then MIN-all-reduces the bytes across ranks.  A rank with no
 * candidates writes all ones (it does not constrain the intersection).
 * Replaces the set building of common_suffix_steps: utils/step_windows.py:22-27. */
int tml_win_presence(tml_ctx* ctx, uint32_t kind, uint64_t glo, uint64_t span,
                     uint8_t* presence_dev, void* stream);

typedef struct tml_align_info {
  uint64_t n_common;    /* aligned steps (<= window)                          */
  uint64_t start_step;
  uint64_t end_step;
  uint64_t n_rows;      /* this rank's rows inside the aligned window         */
  /* aligned per-rank sums (reporting/sections/step_time/alignment.py:44-91):
   * dl, fwd, bwd, opt, step_cpu(=max(0,traced)), traced, total               */
  double t_sums[7];
  /* aligned memory: sum alloc, sum resv, max alloc, max resv
   * (step_memory/model.py:175,224-246)                                       */
  double m_sums[4];
} tml_align_info;

/* Single-rank bulk path.  With one rank the per-step median and worst ARE the rank's values
 * (diagnostics/step_time/adapters.py:92-139 over one column), so ring -> series is one pass
 * (k_window_fused): the 64-B WindowRows are never written or re-read.  tml_win_peek: how many
 * records the ring retains and how many fall into the last-`window` time window (sizes the series
 * buffer, [16][n_window] doubles).  tml_win_fused: *ok = 1 and `aligned` filled if the window is
 * dense (every row a candidate of both kinds, consecutive step ids; memory window == time
 * window); *ok = 0: use the staged path.  Per-rank sums are the deterministic tree sums: a single
 * rank has no tie to break (rel <= 1e-13 of the reference-order sums).                    */
int tml_win_peek(tml_ctx* ctx, uint32_t window, uint64_t* n_retained, uint64_t* n_window);
int tml_win_fused(tml_ctx* ctx, uint32_t window, double* series, void* stream, tml_win_info* out,
                  tml_align_info* aligned, uint32_t* ok);


/* Stage 3 (local, identical on every rank given the reduced presence).
 * Prefix-scan of the common-step flags, keep the last `window`, gather this
 * rank's rows for them into the dense exchange buffer (tml_win_rows) and
 * reduce the per-rank sums.  Replaces common_suffix_steps' sort + suffix and
 * _summary_from_step_metrics: utils/step_windows.py:28-33,
 * step_time/alignment.py:44-155, step_memory/loader.py:208-254. */
int tml_win_select(tml_ctx* ctx, uint32_t kind, uint64_t glo, uint64_t span,
                   const uint8_t* presence_dev, uint32_t window, void* stream,
                   tml_align_info* out);

/* Stage 2+3 shortcut for the lock-step case: when every participating rank's
 * window is dense (tml_win_info.dense) the common window is simply the last W
 * step ids of [max lo, min hi]; no presence map or scan is needed, the aligned
 * rows are a contiguous slice of the window rows.  Same outputs as
 * tml_win_select. */
int tml_win_select_dense(tml_ctx* ctx, uint32_t kind, uint64_t first_step,
                         uint64_t n_common, void* stream, tml_align_info* out);

/* Device pointer / byte size of this rank's aligned rows (n_common x 64 B),
 * valid until the next tml_win_select of the same kind. */
const void* tml_win_rows(tml_ctx* ctx, uint32_t kind);
/* CUDA-IPC export / import of that buffer, for the fused NVLink exchange
 * (peer loads inside tml_win_reduce instead of an NCCL all-gather).  The handle
 * names the allocation the rows live in; the rows start byte_offset into it. */
int tml_win_rows_export(tml_ctx* ctx, uint32_t kind, void* handle64, uint64_t* byte_offset);
int tml_peer_open(tml_ctx* ctx, const void* handle64, void** peer_ptr);
int tml_peer_close(tml_ctx* ctx, void* peer_ptr);

#define TML_SERIES_PER_STEP 16u /* 8 metrics x {median, worst} */
/* series index = metric * 2 + {0 median, 1 worst}; metric order:
 * dataloader_fetch, forward, backward, optimizer_step, step_time(traced),
 * wait_proxy, peak_allocated, peak_reserved                                 */

#define TML_MASK_TIME 1u
#define TML_MASK_MEM 2u

typedef struct tml_reduce_args {
  uint32_t n_ranks;      /* R rows pointers below                            */
  uint32_t mask;         /* TML_MASK_TIME | TML_MASK_MEM                     */
  uint64_t n_common;     /* series length (row count of every rows[r])       */
  uint64_t shard_lo;     /* this call computes steps [shard_lo, shard_hi)    */
  uint64_t shard_hi;
  const void* rows[TML_MAX_RANKS]; /* device ptrs: local, peer-mapped or gathered */
  double* series;        /* device, [16][n_common] f64, caller-allocated     */
} tml_reduce_args;

/* Stage 4.  Per aligned step: derive compute/traced/wait per rank, sort the R
 * values of each metric in registers, write median and max series.  Reads the
 * R x n x 64 B rows exactly once (local HBM or NVLink peer loads).  Replaces
 * _build_metric_series and build_combined_metrics_from_window's per-step
 * columns: diagnostics/step_time/adapters.py:92-139,
 * reporting/sections/step_memory/model.py:141-176. */
int tml_win_reduce(tml_ctx* ctx, const tml_reduce_args* args, void* stream);
/* Device time (ms, CUDA events on the launching stream) of the last k_window_rows
 * (which = 0) / k_window_reduce (which = 1) launch; -1 if none or not finished.
 * Timeline of the last reduce, ms since k_window_rows began: which = 2 the reduce kernel's
 * launch point, 3 the end of the deferred exact sums (side stream), 4 the reduce kernel's end. */
double tml_kernel_ms(tml_ctx* ctx, uint32_t which);

typedef struct tml_band_args {
  uint64_t n_common;
  uint64_t shard_lo, shard_hi;       /* series columns valid on this rank    */
  uint64_t band_lo[2][3];            /* [kind][baseline, mid, recent] ranges */
  uint64_t band_hi[2][3];            /*   in global series index, hi excl.   */
  uint64_t tail_first[2];            /* index of the growth tail's first pt  */
} tml_band_args;

typedef struct tml_band_out {
  double sum[TML_SERIES_PER_STEP][3];   /* partial sums over band ^ shard     */
  uint64_t cnt[TML_SERIES_PER_STEP][3];
  double tail_first[TML_SERIES_PER_STEP]; /* NaN if not on this shard         */
  double tail_last[TML_SERIES_PER_STEP];
} tml_band_out;

/* Stage 5.  Band sums of the series for the trend engines
 * (analytics/trends/core.py:51-115). */
int tml_win_bands(tml_ctx* ctx, const double* series, const tml_band_args* args,
                  void* stream, tml_band_out* out);

typedef struct tml_proc_agg {
  uint64_t n;          /* rows in the window (last max_rows)                 */
  uint64_t n_gpu;      /* rows carrying GPU metrics                          */
  double ts_min, ts_max;
  double sum_cpu, max_cpu;
  double sum_rss, max_rss;
  double sum_used, max_used;
  double sum_resv, max_resv;
  double max_total;
  double max_ratio;    /* MAX(resv / used) over rows with used > 0, else -1  */
  uint32_t max_cores;
  uint32_t any_gpu_available; /* 0/1, valid if n > 0                         */
  double sum_cpu_lo;   /* low word of the double-double cpu sum: the exact sum
                          is sum_cpu + sum_cpu_lo (matches SQLite's compensated
                          AVG to the last bit)                               */
} tml_proc_agg;

/* Per-rank process aggregates over the last max_rows proc records.  Replaces
 * the SQL aggregates of reporting/sections/process/loader.py:56-230. */
int tml_proc_reduce(tml_ctx* ctx, uint32_t max_rows, void* stream,
                    tml_proc_agg* out);
/* Split form: launch without synchronising; collect waits (on an event) only if
 * the results have not landed yet -- normally a later synchronisation of the same
 * stream (tml_win_prepare's) has already covered it. */
int tml_proc_reduce_launch(tml_ctx* ctx, uint32_t max_rows, void* stream);
int tml_proc_reduce_collect(tml_ctx* ctx, tml_proc_agg* out);

/* ---------------------------------------------------------------- WHOLE REDUCE
 * The staged reduce above, sequenced natively for the production layout (one rank
 * per process / GPU): prepare -> bounds exchange (+ process aggregates + the
 * lock-step speculative alignment) -> alignment -> row exchange fused into K4
 * (peer loads) or step-sharded NCCL send/recv -> K4 -> trend bands -> band
 * exchange.  Replaces, for one call of final_summary(), the load + align + reduce
 * half of StepTimeSummarySection / StepMemorySummarySection / ProcessSummarySection
 * (reporting/sections/{step_time,step_memory,process}/__init__.py:50-112); the
 * rank-level rules are then one tml_diag_* call each.
 * The collectives are NCCL calls on the communicator the host side hands in (the
 * training job's own: torch.distributed's ncclComm_t), issued on `stream`.       */
typedef struct tml_comm {
  void* nccl_comm;   /* ncclComm_t spanning the job's ranks; NULL when world == 1 */
  int32_t rank;
  int32_t world;
} tml_comm;

#define TML_XCHG_AUTO 0u  /* peer loads for large / repeated windows, else send-recv */
#define TML_XCHG_P2P 1u   /* CUDA-IPC peer loads fused into K4                      */
#define TML_XCHG_A2A 2u   /* step-sharded ncclSend/ncclRecv, K4 on the received shard */
#define TML_XCHG_LOCAL 3u /* world == 1 (reported, not requested)                    */

typedef struct tml_reduce_run_args {
  uint32_t window;      /* max_rows / window_size of the sections                 */
  uint32_t proc_rows;   /* max process rows (0: skip the process aggregates)      */
  uint32_t exchange;    /* TML_XCHG_*                                             */
  uint32_t speculate;   /* 1: lock-step speculation (alignment rides exchange #1) */
} tml_reduce_run_args;

typedef struct tml_kind_result {
  uint32_t observed;                 /* ranks that had candidates                 */
  uint32_t n_used;                   /* ranks with rows in the aligned window     */
  int32_t used[TML_MAX_RANKS];       /* ascending                                 */
  uint64_t n_common, start_step, end_step;
  uint64_t n_rows[TML_MAX_RANKS];    /* by position in used[]                     */
  double t_sums[TML_MAX_RANKS][7];
  double m_sums[TML_MAX_RANKS][4];
  uint32_t has_bands;
  uint32_t _pad;
  double band_sum[TML_SERIES_PER_STEP][3];   /* summed over ranks, rank order     */
  uint64_t band_cnt[TML_SERIES_PER_STEP][3];
  double tail_first[TML_SERIES_PER_STEP];
  double tail_last[TML_SERIES_PER_STEP];
  uint64_t shard_lo, shard_hi;       /* this rank's columns of the series         */
  const double* series;              /* device, [16][n_common]; owned by the ctx  */
} tml_kind_result;

typedef struct tml_reduce_run_out {
  uint32_t n_ranks;
  uint32_t exchange_used;            /* TML_XCHG_*                                */
  uint32_t fused_pass;               /* time and memory shared one K4 pass        */
  uint32_t n_exchanges;              /* small vector exchanges issued             */
  tml_win_info infos[TML_MAX_RANKS];
  tml_proc_agg procs[TML_MAX_RANKS];
  tml_kind_result time, mem;
  double k3a_ms, k4_ms;              /* device time of the two bandwidth kernels  */
  double stage_ms[5];                /* host clock: prepare, align, reduce (launch), bands, total */
} tml_reduce_run_out;

int tml_reduce_run(tml_ctx* ctx, const tml_comm* comm, const tml_reduce_run_args* args,
                   void* stream, tml_reduce_run_out* out);

/* sizeof() of an ABI struct by name ("tml_win_info", ...), 0 if unknown: lets a binding
 * verify its mirror of the layouts without compiling C. */
uint64_t tml_struct_size(const char* name);

/* ---------------------------------------------------------------- LIVE TICK
 * The render-tick twins of the window reduce: what the reference's live CLI /
 * dashboard recompute every second from SQLite.
 *   kind TML_KIND_TIME  StepCombinedComputer._compute_impl
 *                       (renderers/step_time/compute.py:129-315)
 *   kind TML_KIND_MEM   build_step_memory_combined_result
 *                       (renderers/step_memory/common.py:215-356)
 * Same staging as the reduce above, over the newest `lookback` ring records:
 *   prepare  -> 64-B rows; candidate = newest row of a step id (time:
 *               compute.py:371-401) / newest row with non-NULL peaks (memory:
 *               common.py:143-178); bounds for the intersection
 *   presence -> bytes over [glo, glo+span); caller MIN-all-reduces them.  Memory
 *               view: a rank with no candidate in range writes all ones -- the
 *               reference drops it from the rank maps (common.py:262-275)
 *   select   -> last `window` common step ids (compute.py:452-470,
 *               common.py:359-397), this rank's rows for them, the six raw phase
 *               sums in ascending step order (compute.py:502-531) and the two
 *               memory peaks (common.py:289)
 *   series   -> per-step median / worst / sum across ranks (compute.py:573-596,
 *               common.py:286-287)
 * Runs on any stream, concurrently with the step path (the ring head is read on
 * the device; nothing here touches the training stream).                      */
typedef struct tml_combined_info {
  uint64_t n_rows;      /* look-back rows read from the ring (any row counts)  */
  uint64_t n_cand;      /* candidate step ids among them                      */
  uint64_t lo, hi;      /* min / max candidate step id (valid if n_cand > 0)  */
  uint64_t latest_step; /* max step id: min over ranks = completed_step       */
  uint64_t first_step;  /* step id of the oldest look-back row                */
  uint32_t truncated;   /* 1: the ring holds older rows than the look-back    */
  uint32_t monotone;
} tml_combined_info;

typedef struct tml_combined_align {
  uint64_t n_common;    /* steps_used (<= window), identical on every rank    */
  uint64_t n_rows;      /* this rank's rows for them (0: it is not in the
                           window -- no rows, or no candidate in range)       */
  double sums[6];       /* dl, h2d, fwd, bwd, opt, step wall (ms)             */
  double peaks[2];      /* max peak_alloc, max peak_resv over the window (B)  */
} tml_combined_align;

int tml_combined_prepare(tml_ctx* ctx, uint32_t kind, uint32_t lookback,
                         void* stream, tml_combined_info* out);
int tml_combined_presence(tml_ctx* ctx, uint32_t kind, uint64_t glo,
                          uint64_t span, uint8_t* presence_dev, void* stream);
int tml_combined_select(tml_ctx* ctx, uint32_t kind, uint64_t glo, uint64_t span,
                        const uint8_t* presence_dev, uint32_t window,
                        void* stream, tml_combined_align* out);
/* this rank's aligned rows (n_common x 64 B, ascending step id), or NULL */
const void* tml_combined_rows(tml_ctx* ctx, uint32_t kind);
/* the n_common aligned step ids -> host buffer (only on a rank with n_rows > 0) */
int tml_combined_steps(tml_ctx* ctx, uint32_t kind, uint64_t* steps_host,
                       uint64_t cap, void* stream);
/* series_dev[(col*3 + k) * n_common + j], k = median, worst, sum, for row columns
 * first_col .. first_col+n_cols (time: 0, 6; memory: 6, 2).  rank_rows = device
 * pointers to every present rank's aligned rows (local, gathered or peer-mapped),
 * in rank order. */
int tml_combined_series(tml_ctx* ctx, const void* const* rank_rows,
                        uint32_t n_ranks, uint64_t n_common, uint32_t first_col,
                        uint32_t n_cols, double* series_dev, void* stream);

/* ---------------------------------------------------------------- DIAGNOSIS
 * Host C++ rule engines (O(R) scalars).  Each writes one UTF-8 JSON object
 * whose keys mirror the reference's DiagnosticResult dataclasses. */

typedef struct tml_rank_means {
  int32_t rank;
  int64_t steps_analyzed;
  double dataloader_ms, forward_ms, backward_ms, optimizer_ms, step_cpu_ms;
} tml_rank_means;

typedef struct tml_trend_in { /* band means of one series; valid = enough points */
  int32_t valid;
  double baseline_avg, mid_avg, recent_avg;
} tml_trend_in;

typedef struct tml_st_diag_in {
  int32_t n_ranks;
  int32_t max_rows;
  int64_t n_common;       /* aligned steps with series (0 = no series)       */
  int64_t completed_step;
  tml_rank_means ranks[TML_MAX_RANKS];
  /* trend of the series the reference would pick (median if multi-rank else
   * worst) for step_time, wait_proxy, dataloader_fetch                       */
  tml_trend_in trend_step, trend_wait, trend_dl;
} tml_st_diag_in;

/* Replaces build_summary_step_diagnosis_result -> build_step_diagnosis_result:
 * diagnostics/step_time/adapters.py:232-355, api.py:313-649, context.py,
 * rules.py, trend.py, policy.py:55-73.  Writes "null" when the reference
 * returns None. */
int tml_diag_step_time(const tml_st_diag_in* in, char* json_out, size_t cap);

typedef struct tml_mem_metric_in {
  int32_t n_ranks;                 /* ranks in the aligned window            */
  int32_t ranks[TML_MAX_RANKS];
  double rank_peak[TML_MAX_RANKS]; /* max over aligned steps per rank        */
  tml_trend_in trend_worst, trend_median;
  int32_t points;                  /* series length                          */
  double tail_first, tail_last;    /* worst series endpoints of the last
                                      min(points, 1000) steps                */
} tml_mem_metric_in;

typedef struct tml_mem_diag_in {
  int64_t steps_used;     /* aligned steps                                   */
  int32_t window_size;
  int64_t completed_step;
  int32_t ranks_seen;     /* ranks with any step-memory row                  */
  double gpu_total_bytes; /* <= 0: unknown                                   */
  int32_t n_metrics;      /* 0 (no data) or 2: [peak_allocated, peak_reserved] */
  tml_mem_metric_in metric[2];
} tml_mem_diag_in;

/* Replaces build_combined_metrics_from_window's rank-level part and
 * build_step_memory_summary_diagnosis_result:
 * reporting/sections/step_memory/model.py:175-219,
 * diagnostics/step_memory/api.py:284-508, adapters.py, rules.py, trend.py:203-277. */
int tml_diag_step_memory(const tml_mem_diag_in* in, char* json_out, size_t cap);

typedef struct tml_proc_diag_in {
  int32_t n_ranks;
  int32_t ranks[TML_MAX_RANKS];
  tml_proc_agg agg[TML_MAX_RANKS];
  double ram_total[TML_MAX_RANKS]; /* psutil.virtual_memory().total per rank */
  int32_t gpu_count[TML_MAX_RANKS];
} tml_proc_diag_in;

/* Replaces load_process_section_data's pooled aggregates + diagnose_process:
 * reporting/sections/process/loader.py:56-230,
 * diagnostics/process/context.py:242-340, rules.py:71-345, api.py:84-118. */
int tml_diag_process(const tml_proc_diag_in* in, char* json_out, size_t cap);

/* ---------------------------------------------------------------- SECTIONS
 * All three sections of one tml_reduce_run as one JSON object
 * {"step_time": {data, diagnosis, global, overview}, "step_memory": {...},
 *  "process": {...}}: per-rank RankStepSummary rows, aligned window, public
 * rollups (reporting/sections/step_time/model.py:77-120,270-498,
 * step_memory/model.py:224-246,322-412) and the three tml_diag_* results --
 * what StepTimeSummarySection / StepMemorySummarySection / ProcessSummarySection
 * hand to their kept payload builders
 * (reporting/sections/{step_time,step_memory,process}/__init__.py:50-112).   */
typedef struct tml_sections_args {
  double ram_total;   /* psutil.virtual_memory().total (single node: per-host constant) */
  int32_t gpu_count;  /* torch.cuda.device_count()                                      */
  uint32_t window;
  uint32_t proc_rows; /* 0: no process aggregates were collected                        */
  uint32_t _pad;
} tml_sections_args;

int tml_sections_json(const tml_reduce_run_out* run, const tml_sections_args* args,
                      char* json_out, size_t cap);

/* ---------------------------------------------------------------- DEEP PROFILE
 * K1 / K2 with a layer-id dimension (SURVEY 8f-4).  Replaces the per-layer CUDA-event pairs,
 * event objects and queues of instrumentation/hooks/layer_forward_time_hooks.py:113-267,
 * layer_backward_time_hooks.py:110-264 and the activation sizes of
 * layer_forward_memory_hooks.py:60-190 / layer_backward_memory_hooks.py; one record per
 * (step, layer) replaces the four Layer*Sampler aggregations
 * (samplers/layer_{forward,backward}_{time,memory}_sampler.py).
 *   tml_layer_init    allocate accumulators + a ring of `steps` x n_layers records
 *   tml_layer_begin   %globaltimer stamp on `stream` -> slot (shares the 64 begin slots of K1)
 *   tml_layer_end     stamp + accumulate (t1 - t0), n_calls and the activation bytes of the call
 *                     into layer `layer`, direction 0 forward / 1 backward
 *   tml_layer_commit  close the step: snapshot every layer's accumulators into the ring
 *   tml_layer_drain   completed steps -> host (own stream; never the training stream)        */
typedef struct tml_layer_record {   /* 48 B per (step, layer) */
  uint64_t step;
  uint64_t fwd_ns, bwd_ns;
  uint32_t fwd_calls, bwd_calls;
  uint64_t fwd_bytes, bwd_bytes;    /* output activation / grad-output bytes, summed over calls */
} tml_layer_record;

int tml_layer_init(tml_ctx* ctx, uint32_t n_layers, uint32_t steps);
int tml_layer_begin(tml_ctx* ctx, void* stream);
int tml_layer_end(tml_ctx* ctx, uint32_t layer, uint32_t direction, int slot, uint64_t bytes, void* stream);
int tml_layer_commit(tml_ctx* ctx, uint64_t step, void* stream);
int tml_layer_drain(tml_ctx* ctx, tml_layer_record* out, uint32_t max_steps, uint32_t* n_steps,
                    uint32_t* n_layers, uint64_t* n_dropped);

/* ---------------------------------------------------------------- TEST HOOK
 * Host emulation of K3e -- the reference-order window sums (``s += x`` per row:
 * reporting/sections/step_time/model.py:262-268, alignment.py:59-75) computed as composed
 * integer maps, csrc/tml_exact_sum.h -- for one chain of non-negative doubles.  Runs the same
 * plan / compose / verified-apply / tile-fallback steps as the kernels, serially, so the CPU
 * suite can fuzz the arithmetic against a plain sequential loop.  ``planned`` = 0 skips the
 * plan (every tile composed under the true exponent); ``slow_rows`` = rows that needed a real
 * dependent add.  Never called by the product.                                           */
int tml_xs_host_sum(const double* x, uint64_t n, int planned, double* out_sum, uint64_t* slow_rows);

#ifdef __cplusplus
}
#endif
#endif /* TRACEML_B200_H_ */
