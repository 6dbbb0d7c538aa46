// tml_engine.cu -- kernels + C-ABI of the GPU-native telemetry engine (H100, sm_90a).
//
// Kernel map (DESIGN.md section 4):
//   K1  k_stamp_begin / k_stamp_end   %globaltimer phase stamps on the training stream
//   K2  k_commit                      in-flight record -> smem -> one 128-B line in the
//                                     HBM ring (+ host-mapped mirror), running stats
//   K5  k_proc_commit                 64-B process sample into the proc ring
//   K3a k_window_rows                 ring -> WindowRow[] (ns->ms), step ids, flags, bounds
//   K3b k_presence                    presence bytes over [glo, glo+span)
//   K3c k_sel_count/k_sel_scan/k_sel_scatter   suffix-select of the last W common steps
//   K3d k_gather                      dense aligned rows + per-rank sums
//   K4  k_window_reduce<R>            per-step cross-rank median/max, 16 series
//   K4b k_bands                       trend band sums
//   K6  k_proc_reduce                 per-rank process aggregates
//
// Nothing here is a dense contraction: no tensor-core path.  Every bulk kernel
// is HBM-bound; accesses are 16-byte vectorised and warp-coalesced, tiles are
// staged through swizzled shared memory where the record layout (AoS, 128 B)
// would otherwise make a warp touch 32 lines per load.

#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>

#include "../../include/traceml_b200.h"
#include "tml_internal.h"

typedef unsigned long long u64;
typedef unsigned int u32;
typedef unsigned char u8;

static_assert(sizeof(tml_step_record) == 128, "StepRecord must be 128 B");
static_assert(sizeof(tml_window_row) == 64, "WindowRow must be 64 B");
static_assert(sizeof(tml_proc_record) == 64, "ProcRecord must be 64 B");

#define TML_N_SLOTS 64u      // begin-timestamp slots (regions in flight)
#define TML_N_EPOCHS 8u      // in-flight accumulator sets (steps in flight)
#define TML_HIST_BINS 256u

// row flags written by k_window_rows
#define RF_USABLE 1u       // some summarised phase > 0  (model.py:188-196)
#define RF_HAS_MEM 2u
#define RF_IN_TIME 4u      // inside the last-W time window
#define RF_CAND_T 8u       // time-alignment candidate: usable, in window, first row of its step id
#define RF_CAND_M 16u      // memory candidate: has_mem and last row of its step id

// ------------------------------------------------------------------ device state

struct DevAcc {
  u64 dur_ns[TML_MAX_PHASES];
  u32 n_calls[TML_MAX_PHASES];
  u32 gpu_mask;
  u32 _pad;
};

struct DevState {
  u64 begin_ts[TML_N_SLOTS];
  DevAcc acc[TML_N_EPOCHS];
  u64 head;       // step records committed
  u64 proc_head;  // proc records committed
  u64 live_sum[TML_MAX_PHASES];
  u64 live_max[TML_MAX_PHASES];
  u32 hist[TML_N_PHASES][TML_HIST_BINS];
  tml_live_stats live;  // running count / sum / worst / median per phase (k_mirror copies it out)
  u64 layer_begin_ts[TML_N_SLOTS];  // deep profile: its own begin slots (hundreds of layer regions
                                    // open and close while ONE phase region stays open)
};

// host-mapped page: written by kernels, read by the sampler thread with no CUDA call
struct HostPage {
  volatile u64 mirror_head;
  volatile u64 pmirror_head;
  tml_live_stats live;
};

struct CommitArgs {
  u64 step;
  double host_ts;
  u64 host_dur[TML_MAX_PHASES];
  u32 host_calls[TML_MAX_PHASES];
  u32 epoch;
  u32 flags;
  u64 peak_alloc;  // c10 allocator peaks of the step (host state: they travel as launch arguments)
  u64 peak_resv;
  u64 seq;         // commit number = ring position (the host counts them)
};

struct WinAcc {  // integer side results of k_window_rows (atomics; order-independent)
  u64 lo[2];
  u64 hi[2];
  u64 ncand[2];
  u64 nrows[2];
  u64 latest_step;
  u64 violations;
  u64 dups;
  u64 t_count;
  u64 n_both;  // rows that are candidates of BOTH kinds (time == memory window test)
  u64 msum[2]; // exact sum of peak_alloc / peak_resv over the window rows (byte counts are integers;
               // the reference's mean is CPython's compensated sum = the correctly rounded exact sum)
};

// ------------------------------------------------------------------ device helpers

__device__ __forceinline__ u64 globaltimer_ns() {
  u64 t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ double shfl_xor_f64(double v, int m) {
  return __shfl_xor_sync(0xffffffffu, v, m);
}
__device__ __forceinline__ double shfl_idx_f64(double v, int src, int width) {
  return __shfl_sync(0xffffffffu, v, src, width);
}

// log-linear histogram bin of a duration: 8 sub-bins per octave, 2^0 .. 2^32 ns
__device__ __forceinline__ u32 hist_bin(u64 ns) {
  if (ns < 8ull) return (u32)ns;
  if (ns >> 32) return TML_HIST_BINS - 1u;
  int msb = 63 - __clzll((long long)ns);  // >= 3
  u32 sub = (u32)((ns >> (msb - 3)) & 7ull);
  return (u32)(msb << 3) | sub;  // msb in [3,31] -> bins 24..255
}
__device__ __forceinline__ u64 hist_bin_center(u32 bin) {
  if (bin < 8u) return (u64)bin;
  u32 msb = bin >> 3, sub = bin & 7u;
  u64 lo = (1ull << msb) + ((u64)sub << (msb - 3));
  return lo + ((1ull << (msb - 3)) >> 1);
}

// ------------------------------------------------------------------ K1: stamps

__global__ void k_stamp_begin(DevState* st, u32 slot) {
  if (threadIdx.x == 0) st->begin_ts[slot] = globaltimer_ns();
}

__global__ void k_stamp_end(DevState* st, u32 slot, u32 phase, u32 epoch) {
  if (threadIdx.x == 0) {
    u64 t1 = globaltimer_ns();
    u64 t0 = st->begin_ts[slot];
    u64 d = (t1 > t0) ? (t1 - t0) : 0ull;
    DevAcc* a = &st->acc[epoch];
    atomicAdd(&a->dur_ns[phase], d);
    atomicAdd(&a->n_calls[phase], 1u);
    atomicOr(&a->gpu_mask, 1u << phase);
  }
}

// ------------------------------------------------------------------ K2: commit
// 6 warps: warp p owns phase p's running statistics; warp 0 also assembles the
// 128-B record in shared memory and writes it as 8 x 16-B coalesced stores.

// Nothing in here leaves the GPU: writing the record and the live statistics into host-mapped
// memory and closing with __threadfence_system would cost the TRAINING stream time every step for
// the benefit of a sampler that looks twice a second.  The sampler instead fetches what it needs itself (k_mirror, on its own stream, tml_drain / tml_live).
__global__ void __launch_bounds__(192) k_commit(DevState* st, tml_step_record* ring, u32 ring_slots,
                                                 CommitArgs a) {
  __shared__ __align__(16) u64 rec[16];
  __shared__ u64 s_dur[TML_MAX_PHASES];
  __shared__ u32 s_calls[TML_MAX_PHASES];
  __shared__ u32 s_mask;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  DevAcc* acc = &st->acc[a.epoch];

  // ONE global round trip on the critical path: the phase accumulator and the 256-bin histogram
  // (8 bins per lane) are fetched together; the +1 of this step is applied in registers and
  // written back without being waited for (instead of accumulator -> histogram RMW -> histogram
  // re-read -> head read: four dependent round trips).
  u32* h = st->hist[warp];
  u32 c[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) c[k] = h[lane * 8 + k];
  u64 dur = 0, run_sum = 0, run_max = 0;
  u32 calls = 0;
  if (lane == 0) {
    dur = acc->dur_ns[warp] + a.host_dur[warp];
    calls = acc->n_calls[warp] + a.host_calls[warp];
    run_sum = st->live_sum[warp];
    run_max = st->live_max[warp];
    s_dur[warp] = dur;
    s_calls[warp] = calls;
    acc->dur_ns[warp] = 0;
    acc->n_calls[warp] = 0;
    if (warp == 0) {
      s_mask = acc->gpu_mask;
      acc->gpu_mask = 0;
      // spare accumulator slots ("other" regions) are reset, not recorded
      acc->dur_ns[6] = 0; acc->dur_ns[7] = 0; acc->n_calls[6] = 0; acc->n_calls[7] = 0;
    }
  }
  dur = __shfl_sync(0xffffffffu, dur, 0);
  calls = __shfl_sync(0xffffffffu, calls, 0);

  // running statistics of phase `warp`: count / sum / worst exactly, median from
  // the log histogram by a warp-shuffle inclusive scan of per-lane bin counts.
  if (calls > 0u) {
    const u32 bin = hist_bin(dur);
    if ((int)(bin >> 3) == lane) {
#pragma unroll
      for (int k = 0; k < 8; ++k) c[k] += ((bin & 7u) == (u32)k) ? 1u : 0u;
      h[bin] = c[0] * ((bin & 7u) == 0u) + c[1] * ((bin & 7u) == 1u) + c[2] * ((bin & 7u) == 2u) +
               c[3] * ((bin & 7u) == 3u) + c[4] * ((bin & 7u) == 4u) + c[5] * ((bin & 7u) == 5u) +
               c[6] * ((bin & 7u) == 6u) + c[7] * ((bin & 7u) == 7u);
    }
    u32 local = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) local += c[k];
    u32 incl = local;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      u32 n = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += n;
    }
    u32 total = __shfl_sync(0xffffffffu, incl, 31);
    u32 target = (total + 1u) >> 1;
    u32 excl = incl - local;
    unsigned hit = __ballot_sync(0xffffffffu, (excl < target) && (target <= incl));
    int src = __ffs(hit) - 1;
    const u64 sum = __shfl_sync(0xffffffffu, run_sum, 0) + dur;
    u64 mx = __shfl_sync(0xffffffffu, run_max, 0);
    mx = dur > mx ? dur : mx;
    if (lane == src) {
      u32 run = excl;
      u32 mbin = lane * 8;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        run += c[k];
        if (run >= target) { mbin = lane * 8 + k; break; }
      }
      st->live_sum[warp] = sum;
      st->live_max[warp] = mx;
      tml_live_phase* lp = &st->live.phase[warp];
      lp->count = total;
      lp->sum_ns = sum;
      lp->worst_ns = mx;
      lp->median_ns = hist_bin_center(mbin);
    }
  }
  __syncthreads();

  if (warp == 0) {
    const u64 seq = a.seq;  // the host counts commits: no read of the head on the critical path
    if (lane == 0) {
      rec[0] = a.step;
#pragma unroll
      for (int p = 0; p < 6; ++p) rec[1 + p] = s_dur[p];
      rec[7] = (u64)s_calls[0] | ((u64)s_calls[1] << 32);
      rec[8] = (u64)s_calls[2] | ((u64)s_calls[3] << 32);
      rec[9] = (u64)s_calls[4] | ((u64)s_calls[5] << 32);
      rec[10] = a.peak_alloc;
      rec[11] = a.peak_resv;
      rec[12] = (u64)__double_as_longlong(a.host_ts);
      rec[13] = (u64)s_mask | ((u64)a.flags << 32);
      rec[14] = seq;
      rec[15] = 0;
    }
    __syncwarp();
    if (lane < 8) {
      uint4 v = reinterpret_cast<const uint4*>(rec)[lane];
      reinterpret_cast<uint4*>(&ring[seq % ring_slots])[lane] = v;
    }
    __syncwarp();
    if (lane == 0) {
      __threadfence();  // the record is visible to every later reader of `head` on this GPU
      st->live.steps_committed = seq + 1;
      st->head = seq + 1;
    }
  }
}

// Sampler side: copy the records committed since `from` (at most the newest mirror_slots) and the
// live statistics into host-mapped memory.  One CTA, on the sampler's own stream; the caller
// synchronises that stream, so no system-scope fence is needed here either.
__global__ void __launch_bounds__(1024) k_mirror(const DevState* st, const tml_step_record* __restrict__ ring,
                                                  u32 ring_slots, tml_step_record* mirror, u32 mirror_slots,
                                                  HostPage* page, u64 from) {
  __shared__ u64 s_head;
  if (threadIdx.x == 0) s_head = *reinterpret_cast<const volatile u64*>(&st->head);
  __syncthreads();
  const u64 head = s_head;
  if (head - from > (u64)mirror_slots) from = head - mirror_slots;
  const u64 n16 = (head - from) * 8ull;  // 16-B pieces
  for (u64 k = threadIdx.x; k < n16; k += blockDim.x) {
    const u64 seq = from + (k >> 3);
    const int q = (int)(k & 7);
    reinterpret_cast<uint4*>(&mirror[seq % mirror_slots])[q] =
        reinterpret_cast<const uint4*>(&ring[seq % ring_slots])[q];
  }
  const int nl = (int)(sizeof(tml_live_stats) / 8);
  for (int k = threadIdx.x; k < nl; k += blockDim.x)
    reinterpret_cast<volatile u64*>(&page->live)[k] = reinterpret_cast<const volatile u64*>(&st->live)[k];
  __syncthreads();
  if (threadIdx.x == 0) page->mirror_head = head;
}

// ------------------------------------------------------------------ K1/K2 with a layer id (deep profile)
struct LayerAcc {
  u64 fwd_ns, bwd_ns, fwd_bytes, bwd_bytes;
  u32 fwd_calls, bwd_calls;
  u32 _pad[2];
};
static_assert(sizeof(LayerAcc) == 48, "LayerAcc");

__global__ void k_layer_begin(DevState* st, u32 slot) {
  if (threadIdx.x == 0) st->layer_begin_ts[slot] = globaltimer_ns();
}

__global__ void k_layer_end(DevState* st, LayerAcc* acc, u32 slot, u32 layer, u32 dir, u64 bytes) {
  if (threadIdx.x == 0) {
    const u64 t1 = globaltimer_ns();
    const u64 t0 = st->layer_begin_ts[slot];
    const u64 d = (t1 > t0) ? (t1 - t0) : 0ull;
    LayerAcc* a = &acc[layer];
    if (dir == 0u) { atomicAdd(&a->fwd_ns, d); atomicAdd(&a->fwd_calls, 1u); atomicAdd(&a->fwd_bytes, bytes); }
    else { atomicAdd(&a->bwd_ns, d); atomicAdd(&a->bwd_calls, 1u); atomicAdd(&a->bwd_bytes, bytes); }
  }
}

// one thread per layer: accumulators -> ring slot of this step (48-B records, coalesced), reset
__global__ void k_layer_commit(LayerAcc* acc, tml_layer_record* ring, u32 n_layers, u32 ring_steps, u64 seq,
                               u64 step, u64* head) {
  const u32 l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < n_layers) {
    LayerAcc a = acc[l];
    tml_layer_record r;
    r.step = step; r.fwd_ns = a.fwd_ns; r.bwd_ns = a.bwd_ns; r.fwd_calls = a.fwd_calls; r.bwd_calls = a.bwd_calls;
    r.fwd_bytes = a.fwd_bytes; r.bwd_bytes = a.bwd_bytes;
    ring[(size_t)(seq % ring_steps) * n_layers + l] = r;
    LayerAcc z;
    memset(&z, 0, sizeof(z));
    acc[l] = z;
  }
  __syncthreads();
  if (gridDim.x == 1) {
    if (threadIdx.x == 0) { __threadfence(); *head = seq + 1; }
  }
}
__global__ void k_layer_head(u64* head, u64 v) { *head = v; }

// ------------------------------------------------------------------ K5: proc commit

__global__ void k_proc_commit(DevState* st, tml_proc_record* ring, u32 slots,
                              tml_proc_record* mirror, u32 mirror_slots, HostPage* page,
                              tml_proc_record r) {
  __shared__ __align__(16) tml_proc_record s;
  const int lane = threadIdx.x;
  u64 seq = 0;
  if (lane == 0) { s = r; seq = st->proc_head; }
  seq = __shfl_sync(0xffffffffu, seq, 0);
  __syncwarp();
  if (lane < 4) {
    uint4 v = reinterpret_cast<const uint4*>(&s)[lane];
    reinterpret_cast<uint4*>(&ring[seq % slots])[lane] = v;
    reinterpret_cast<uint4*>(&mirror[seq % mirror_slots])[lane] = v;
  }
  __syncwarp();
  if (lane == 0) {
    __threadfence_system();
    st->proc_head = seq + 1;
    page->pmirror_head = seq + 1;
  }
}

// ------------------------------------------------------------------ reductions

// Deterministic block sum of NV values per thread -> out[NV] (thread 0 writes).
template <int NV, int NTHREADS>
__device__ __forceinline__ void block_sum(double (&v)[NV], double* out) {
  __shared__ double s_part[NTHREADS / 32][NV];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double x = v[k];
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) x += shfl_xor_f64(x, m);
    if (lane == 0) s_part[warp][k] = x;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double x = 0.0;
#pragma unroll
    for (int w = 0; w < NTHREADS / 32; ++w) x += s_part[w][threadIdx.x];
    out[threadIdx.x] = x;
  }
  __syncthreads();
}

// out[c] = reduce over b of partials[b * ncols + c]; op per column: 0 sum, 1 max.
// One warp per column: lane l folds blocks l, l+32, ... in order, then a fixed
// shuffle tree -- deterministic for a given grid, and ~nblk/32 dependent loads deep.
__global__ void k_finalize(const double* __restrict__ partials, int nblk, int ncols, u32 max_mask,
                           double* __restrict__ out) {
  const int c = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (c >= ncols) return;
  const bool is_max = (max_mask >> c) & 1u;
  double x = is_max ? -INFINITY : 0.0;
  for (int b = lane; b < nblk; b += 32) {
    double p = partials[(size_t)b * ncols + c];
    x = is_max ? fmax(x, p) : (x + p);
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    double y = shfl_xor_f64(x, m);
    x = is_max ? fmax(x, y) : (x + y);
  }
  if (lane == 0) out[c] = x;
}

// ------------------------------------------------------------------ K3a: window rows
// Ring (128-B AoS records) -> WindowRow[] (64 B), step ids, row flags, bounds, sums.
//   * tiles are fetched with cp.async (LDGSTS, 16 B per lane per copy, fully coalesced)
//     into XOR-swizzled shared buffers, two per warp, so tile i+1 is in flight while
//     tile i is converted -- without it the kernel is HBM-latency-bound (long-scoreboard
//     stalls);
//   * the swizzle makes the per-lane 128-B record read bank-conflict-free;
//   * rows leave through a swizzled staging buffer as coalesced 16-B stores;
//   * integer side results live in registers for the whole persistent loop.

// ns -> ms as the CORRECTLY ROUNDED quotient ns / 1e6 (what Python's ns / 1e6 gives)
// without a division: y = RN(1/1e6), q = RN(a*y), r = a - 1e6*q (exact, FMA),
// result = RN(q + r*y) -- Markstein's final division step, exact because y is the
// correctly rounded reciprocal (tests/test_ns_to_ms_cpu.py; 2*10^9 values checked once).
__device__ __forceinline__ double ns_to_ms(u64 ns) {
  const double a = (double)ns;
  const double y = 1.0e-6;
  const double q = __dmul_rn(a, y);
  const double r = __fma_rn(-1.0e6, q, a);
  return __fma_rn(r, y, q);
}

#define WR_THREADS 256
#define WR_WARPS (WR_THREADS / 32)
// per warp: two 32-record input buffers (2 x 4 KB) + one 32-row output buffer (2 KB)
#define WR_WARP_U4 (2 * 32 * 8 + 32 * 4)
#define WR_SMEM_BYTES (WR_WARPS * WR_WARP_U4 * 16)

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// one warp fetches its 32-record tile: 8 x cp.async per lane, each instruction = 512 B contiguous.
// slot0 = ring slot of the tile's first record (maintained incrementally by the caller).
__device__ __forceinline__ void wr_issue_warp(uint4* buf, const uint4* __restrict__ ring4, u32 ring_slots,
                                              u64 slot0, u64 n, u64 base, int lane) {
  if (base + 32 <= n && slot0 + 32 <= (u64)ring_slots) {  // whole tile, no ring wrap: linear addresses
    const uint4* src = ring4 + slot0 * 8;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int idx = c * 32 + lane;
      cp_async16(&buf[(idx & ~7) | ((idx ^ (idx >> 3)) & 7)], src + idx);
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int idx = c * 32 + lane;
    const int r = idx >> 3, q = idx & 7;
    if (base + (u64)r < n) {
      u64 slot = slot0 + (u64)r;
      while (slot >= ring_slots) slot -= ring_slots;
      cp_async16(&buf[r * 8 + (q ^ (r & 7))], &ring4[slot * 8 + q]);
    }
  }
}

// K3a.  Persistent grid, WARP-PRIVATE software pipelines: every warp streams its own
// 32-record tiles (cp.async double buffer -> XOR-swizzled smem -> registers -> swizzled
// smem -> coalesced 16-B stores) and synchronises only with __syncwarp; neighbour step
// ids come from warp shuffles (tile edges: two 8-B global reads).  No block barrier in
// the loop (block barriers and waits dominate once the loads are asynchronous).
__global__ void __launch_bounds__(WR_THREADS, 2) k_window_rows(
    const tml_step_record* __restrict__ ring, u32 ring_slots, u64 first_k, u64 n, u64 t_start,
    tml_window_row* __restrict__ rows, u64* __restrict__ steps, u8* __restrict__ flags,
    WinAcc* acc, double* partials, double* __restrict__ csum, u64 csum_top) {
  extern __shared__ __align__(16) unsigned char wr_smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint4* w_in0 = reinterpret_cast<uint4*>(wr_smem) + warp * WR_WARP_U4;
  uint4* w_in1 = w_in0 + 32 * 8;
  uint4* w_out = w_in1 + 32 * 8;

  u64 a_lo0 = ~0ull, a_lo1 = ~0ull, a_hi0 = 0, a_hi1 = 0, a_latest = 0;
  u32 a_nc0 = 0, a_nc1 = 0, a_nr0 = 0, a_nr1 = 0, a_viol = 0, a_dups = 0, a_tc = 0, a_both = 0;
  u64 a_sa = 0, a_sr = 0;                        // exact integer byte sums (window rows)
  double sums[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};  // 7 time sums (tree order) + 2 unused columns
  double mx_a = -INFINITY, mx_r = -INFINITY;      // rank peaks over the window rows
  const u64 nwt = (n + 31) / 32;
  const u64 wstride = (u64)gridDim.x * WR_WARPS;
  const uint4* ring4 = reinterpret_cast<const uint4*>(ring);
  uint4* rows4 = reinterpret_cast<uint4*>(rows);

  u64 wt = (u64)blockIdx.x * WR_WARPS + warp;
  // ring slot of this warp's current tile and the per-trip advance, both kept < ring_slots:
  // two 64-bit modulos per warp for the whole kernel instead of one per lane per tile
  u64 slot_cur = (first_k + wt * 32) % ring_slots;
  const u64 slot_adv = (wstride * 32) % ring_slots;
  if (wt < nwt) wr_issue_warp(w_in0, ring4, ring_slots, slot_cur, n, wt * 32, lane);
  cp_async_commit();

  for (int it = 0; wt < nwt; wt += wstride, ++it) {
    uint4* cur = (it & 1) ? w_in1 : w_in0;
    uint4* nxt = (it & 1) ? w_in0 : w_in1;
    const u64 base = wt * 32;
    const u64 next = wt + wstride;
    u64 slot_next = slot_cur + slot_adv;
    if (slot_next >= ring_slots) slot_next -= ring_slots;
    if (next < nwt) wr_issue_warp(nxt, ring4, ring_slots, slot_next, n, next * 32, lane);
    cp_async_commit();
    // tile-edge neighbours (first/last-of-step tests) straight from the ring
    u64 halo_step = 0;
    u32 halo_flags = 0;
    if (lane == 0 && base > 0) halo_step = ring[slot_cur == 0 ? ring_slots - 1 : slot_cur - 1].step;
    if (lane == 31 && base + 32 < n) {
      u64 hs = slot_cur + 32;
      while (hs >= ring_slots) hs -= ring_slots;
      const tml_step_record* p = &ring[hs];
      halo_step = p->step; halo_flags = p->flags;
    }
    slot_cur = slot_next;
    cp_async_wait<1>();  // this tile has landed; the next one stays in flight
    __syncwarp();

    const u64 i = base + (u64)lane;
    const bool live = i < n;
    const int sw = lane & 7;
    const uint4 c0 = cur[lane * 8 + (0 ^ sw)], c1 = cur[lane * 8 + (1 ^ sw)];
    const uint4 c2 = cur[lane * 8 + (2 ^ sw)], c3 = cur[lane * 8 + (3 ^ sw)];
    const uint4 c5 = cur[lane * 8 + (5 ^ sw)], c6 = cur[lane * 8 + (6 ^ sw)];
    const u64 step = (u64)c0.x | ((u64)c0.y << 32);
    const u32 rflags = c6.w;
    u64 prev_step = __shfl_up_sync(0xffffffffu, step, 1);
    u64 next_step = __shfl_down_sync(0xffffffffu, step, 1);
    u32 next_flags = __shfl_down_sync(0xffffffffu, rflags, 1);
    if (lane == 0) prev_step = halo_step;
    if (lane == 31) { next_step = halo_step; next_flags = halo_flags; }
    double t_dl = 0.0, t_fwd = 0.0, t_bwd = 0.0, t_opt = 0.0, t_wall = 0.0, t_tr = 0.0;  // K3e chunk sums

    if (live) {
      const u64 d0 = (u64)c0.z | ((u64)c0.w << 32);
      const u64 d1 = (u64)c1.x | ((u64)c1.y << 32);
      const u64 d2 = (u64)c1.z | ((u64)c1.w << 32);
      const u64 d3 = (u64)c2.x | ((u64)c2.y << 32);
      const u64 d4 = (u64)c2.z | ((u64)c2.w << 32);
      const u64 d5 = (u64)c3.x | ((u64)c3.y << 32);
      const u64 pa = (u64)c5.x | ((u64)c5.y << 32);
      const u64 pr = (u64)c5.z | ((u64)c5.w << 32);
      const double dl = ns_to_ms(d0), h2d = ns_to_ms(d1), fwd = ns_to_ms(d2);
      const double bwd = ns_to_ms(d3), opt = ns_to_ms(d4), wall = ns_to_ms(d5);
      const bool has_mem = (rflags & TML_REC_HAS_MEM) != 0u;
      const bool usable = (dl > 0.0) || (fwd > 0.0) || (bwd > 0.0) || (opt > 0.0) || (wall > 0.0);
      const bool in_time = i >= t_start;
      const bool uit = usable && in_time;
      const bool has_prev = i > 0, has_next = (i + 1) < n;
      const bool first_in_win = (i == t_start) || !has_prev || (prev_step != step);
      const bool last_m = !has_next || (next_step != step) || ((next_flags & TML_REC_HAS_MEM) == 0u);
      u8 f = 0;
      if (usable) f |= RF_USABLE;
      if (has_mem) f |= RF_HAS_MEM;
      if (in_time) f |= RF_IN_TIME;
      const bool cand_t = usable && in_time && first_in_win;
      const bool cand_m = has_mem && last_m;
      if (cand_t) f |= RF_CAND_T;
      if (cand_m) f |= RF_CAND_M;
      steps[i] = step;
      flags[i] = f;

      a_latest = step > a_latest ? step : a_latest;
      a_viol += (has_prev && step < prev_step) ? 1u : 0u;
      a_dups += (has_prev && step == prev_step) ? 1u : 0u;
      a_nr0 += in_time ? 1u : 0u;
      a_nr1 += has_mem ? 1u : 0u;
      if (cand_t) { a_lo0 = step < a_lo0 ? step : a_lo0; a_hi0 = step > a_hi0 ? step : a_hi0; ++a_nc0; }
      if (cand_m) { a_lo1 = step < a_lo1 ? step : a_lo1; a_hi1 = step > a_hi1 ? step : a_hi1; ++a_nc1; }
      a_both += (cand_t && cand_m) ? 1u : 0u;

      if (usable && in_time) {  // model.py:241-271, same expression order
        const double compute = (fwd + bwd) + opt;
        const double traced = fmax(wall, compute);
        sums[0] += dl; sums[1] += fwd; sums[2] += bwd; sums[3] += opt;
        sums[4] += wall; sums[5] += traced; sums[6] += dl + traced;
        ++a_tc;
      }
      if (in_time) {
        a_sa += pa; a_sr += pr;
        mx_a = fmax(mx_a, (double)pa); mx_r = fmax(mx_r, (double)pr);
      }

      if (csum) { t_dl = uit ? dl : 0.0; t_fwd = uit ? fwd : 0.0; t_bwd = uit ? bwd : 0.0; t_opt = uit ? opt : 0.0;
                  t_wall = uit ? wall : 0.0; t_tr = uit ? fmax(wall, (fwd + bwd) + opt) : 0.0; }

      // row -> swizzled staging (4 x 16 B)
      double2 o0 = make_double2(dl, h2d), o1 = make_double2(fwd, bwd);
      double2 o2 = make_double2(opt, wall), o3 = make_double2((double)pa, (double)pr);
      const int so = (lane >> 1) & 3;
      w_out[lane * 4 + (0 ^ so)] = *reinterpret_cast<uint4*>(&o0);
      w_out[lane * 4 + (1 ^ so)] = *reinterpret_cast<uint4*>(&o1);
      w_out[lane * 4 + (2 ^ so)] = *reinterpret_cast<uint4*>(&o2);
      w_out[lane * 4 + (3 ^ so)] = *reinterpret_cast<uint4*>(&o3);
    }
    if (csum) {
      // approximate sums of this 32-row tile for K3e's plan (any order will do: they only choose the
      // exponent a chunk is composed under, and that choice is verified when the map is applied).
      // The tile lies inside ONE 256-row chunk because chunks are aligned to row indices.
      // Transposed butterfly: 8 values per lane -> 4 -> 2 -> 1 while the lanes pair up over bits
      // 4, 3, 2 (each lane passes on the half it does not keep), then two plain levels over bits
      // 1, 0: 9 exchanges instead of 35.  Lane 4 j ends up with the tile total of value j.
      double v[8] = {t_dl, t_fwd, t_bwd, t_opt, t_wall, t_tr, t_dl + t_tr, 0.0};
      {
        const bool hi = (lane & 16) != 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const double keep = hi ? v[i + 4] : v[i], send = hi ? v[i] : v[i + 4];
          v[i] = keep + shfl_xor_f64(send, 16);
        }
      }
      {
        const bool hi = (lane & 8) != 0;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const double keep = hi ? v[i + 2] : v[i], send = hi ? v[i] : v[i + 2];
          v[i] = keep + shfl_xor_f64(send, 8);
        }
      }
      {
        const bool hi = (lane & 4) != 0;
        const double keep = hi ? v[1] : v[0], send = hi ? v[0] : v[1];
        v[0] = keep + shfl_xor_f64(send, 4);
      }
      v[0] += shfl_xor_f64(v[0], 2);
      v[0] += shfl_xor_f64(v[0], 1);
      if (base <= csum_top) {
        double* dst = csum + ((csum_top - base) >> 8) * 8;
        if ((lane & 3) == 0 && lane < 28 && v[0] != 0.0) atomicAdd(dst + (lane >> 2), v[0]);
      }
    }
    __syncwarp();
    if (base + 32 <= n) {
      uint4* dst = rows4 + base * 4;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int idx = c * 32 + lane;
        dst[idx] = w_out[(idx & ~3) | ((idx ^ (idx >> 3)) & 3)];
      }
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int idx = c * 32 + lane;
        const int r = idx >> 2, q = idx & 3;
        const u64 ii = base + (u64)r;
        if (ii < n) rows4[ii * 4 + q] = w_out[r * 4 + (q ^ ((r >> 1) & 3))];
      }
    }
    __syncwarp();  // w_out and `cur` are free again
  }
  cp_async_wait<0>();
  {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      u64 t;
      t = __shfl_xor_sync(0xffffffffu, a_lo0, m); a_lo0 = t < a_lo0 ? t : a_lo0;
      t = __shfl_xor_sync(0xffffffffu, a_lo1, m); a_lo1 = t < a_lo1 ? t : a_lo1;
      t = __shfl_xor_sync(0xffffffffu, a_hi0, m); a_hi0 = t > a_hi0 ? t : a_hi0;
      t = __shfl_xor_sync(0xffffffffu, a_hi1, m); a_hi1 = t > a_hi1 ? t : a_hi1;
      t = __shfl_xor_sync(0xffffffffu, a_latest, m); a_latest = t > a_latest ? t : a_latest;
      a_sa += __shfl_xor_sync(0xffffffffu, a_sa, m); a_sr += __shfl_xor_sync(0xffffffffu, a_sr, m);
    }
    a_nc0 = __reduce_add_sync(0xffffffffu, a_nc0); a_nc1 = __reduce_add_sync(0xffffffffu, a_nc1);
    a_nr0 = __reduce_add_sync(0xffffffffu, a_nr0); a_nr1 = __reduce_add_sync(0xffffffffu, a_nr1);
    a_viol = __reduce_add_sync(0xffffffffu, a_viol); a_dups = __reduce_add_sync(0xffffffffu, a_dups);
    a_tc = __reduce_add_sync(0xffffffffu, a_tc); a_both = __reduce_add_sync(0xffffffffu, a_both);
    if (lane == 0) {
      if (a_nc0) { atomicMin(&acc->lo[0], a_lo0); atomicMax(&acc->hi[0], a_hi0); atomicAdd(&acc->ncand[0], (u64)a_nc0); }
      if (a_nc1) { atomicMin(&acc->lo[1], a_lo1); atomicMax(&acc->hi[1], a_hi1); atomicAdd(&acc->ncand[1], (u64)a_nc1); }
      if (a_nr0) atomicAdd(&acc->nrows[0], (u64)a_nr0);
      if (a_nr1) atomicAdd(&acc->nrows[1], (u64)a_nr1);
      atomicMax(&acc->latest_step, a_latest);
      if (a_viol) atomicAdd(&acc->violations, (u64)a_viol);
      if (a_dups) atomicAdd(&acc->dups, (u64)a_dups);
      if (a_tc) atomicAdd(&acc->t_count, (u64)a_tc);
      if (a_both) atomicAdd(&acc->n_both, (u64)a_both);
      if (a_sa) atomicAdd(&acc->msum[0], a_sa);
      if (a_sr) atomicAdd(&acc->msum[1], a_sr);
    }
  }
  __syncthreads();
  block_sum<9, WR_THREADS>(sums, partials + (size_t)blockIdx.x * 11);
  {  // the two maxima: warp shuffle + shared memory, written as partial columns 9, 10
    __shared__ double s_mx[WR_THREADS / 32][2];
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      mx_a = fmax(mx_a, shfl_xor_f64(mx_a, m));
      mx_r = fmax(mx_r, shfl_xor_f64(mx_r, m));
    }
    if (lane == 0) { s_mx[warp][0] = mx_a; s_mx[warp][1] = mx_r; }
    __syncthreads();
    if (tid < 2) {
      double x = -INFINITY;
      for (int w = 0; w < WR_THREADS / 32; ++w) x = fmax(x, s_mx[w][tid]);
      partials[(size_t)blockIdx.x * 11 + 9 + tid] = x;
    }
  }
}



// ------------------------------------------------------------------ K3a+K4 fused (single rank)
// With ONE rank the cross-rank median and worst of a step are the rank's own value, so the
// per-step series can be written straight from the ring records: 128 B in, 128 B out per step, and
// the 64-B WindowRows -- written by K3a only to be re-read by K4 (256 MB each way at
// W = 4e6) -- never exist.  Same warp-private
// cp.async pipeline as k_window_rows; lane = record, so each of the 16 series receives 32
// consecutive doubles per tile: 256-B fully coalesced stores, no staging buffer.  Bounds, counters,
// tree sums and maxima are produced exactly as in k_window_rows; the host accepts the series only
// if the window turns out dense (every row a candidate of both kinds, consecutive step ids),
// otherwise it falls back to the staged path.
#define WF_WARP_U4 (2 * 32 * 8)
#define WF_SMEM_BYTES (WR_WARPS * WF_WARP_U4 * 16)

__global__ void __launch_bounds__(WR_THREADS, 2) k_window_fused(
    const tml_step_record* __restrict__ ring, u32 ring_slots, u64 first_k, u64 n, u64 t_start,
    double* __restrict__ series, u64 n_ser, WinAcc* acc, double* partials) {
  extern __shared__ __align__(16) unsigned char wr_smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint4* w_in0 = reinterpret_cast<uint4*>(wr_smem) + warp * WF_WARP_U4;
  uint4* w_in1 = w_in0 + 32 * 8;

  u64 a_lo0 = ~0ull, a_lo1 = ~0ull, a_hi0 = 0, a_hi1 = 0, a_latest = 0;
  u32 a_nc0 = 0, a_nc1 = 0, a_nr0 = 0, a_nr1 = 0, a_viol = 0, a_dups = 0, a_tc = 0, a_both = 0;
  u64 a_sa = 0, a_sr = 0;
  double sums[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  double mx_a = -INFINITY, mx_r = -INFINITY;
  const u64 nwt = (n + 31) / 32;
  const u64 wstride = (u64)gridDim.x * WR_WARPS;
  const uint4* ring4 = reinterpret_cast<const uint4*>(ring);

  u64 wt = (u64)blockIdx.x * WR_WARPS + warp;
  u64 slot_cur = (first_k + wt * 32) % ring_slots;
  const u64 slot_adv = (wstride * 32) % ring_slots;
  if (wt < nwt) wr_issue_warp(w_in0, ring4, ring_slots, slot_cur, n, wt * 32, lane);
  cp_async_commit();

  for (int it = 0; wt < nwt; wt += wstride, ++it) {
    uint4* cur = (it & 1) ? w_in1 : w_in0;
    uint4* nxt = (it & 1) ? w_in0 : w_in1;
    const u64 base = wt * 32;
    const u64 next = wt + wstride;
    u64 slot_next = slot_cur + slot_adv;
    if (slot_next >= ring_slots) slot_next -= ring_slots;
    if (next < nwt) wr_issue_warp(nxt, ring4, ring_slots, slot_next, n, next * 32, lane);
    cp_async_commit();
    u64 halo_step = 0;
    u32 halo_flags = 0;
    if (lane == 0 && base > 0) halo_step = ring[slot_cur == 0 ? ring_slots - 1 : slot_cur - 1].step;
    if (lane == 31 && base + 32 < n) {
      u64 hs = slot_cur + 32;
      while (hs >= ring_slots) hs -= ring_slots;
      const tml_step_record* p = &ring[hs];
      halo_step = p->step; halo_flags = p->flags;
    }
    slot_cur = slot_next;
    cp_async_wait<1>();
    __syncwarp();

    const u64 i = base + (u64)lane;
    const bool live = i < n;
    const int sw = lane & 7;
    const uint4 c0 = cur[lane * 8 + (0 ^ sw)], c1 = cur[lane * 8 + (1 ^ sw)];
    const uint4 c2 = cur[lane * 8 + (2 ^ sw)], c3 = cur[lane * 8 + (3 ^ sw)];
    const uint4 c5 = cur[lane * 8 + (5 ^ sw)], c6 = cur[lane * 8 + (6 ^ sw)];
    const u64 step = (u64)c0.x | ((u64)c0.y << 32);
    const u32 rflags = c6.w;
    u64 prev_step = __shfl_up_sync(0xffffffffu, step, 1);
    u64 next_step = __shfl_down_sync(0xffffffffu, step, 1);
    u32 next_flags = __shfl_down_sync(0xffffffffu, rflags, 1);
    if (lane == 0) prev_step = halo_step;
    if (lane == 31) { next_step = halo_step; next_flags = halo_flags; }

    if (live) {
      const u64 d0 = (u64)c0.z | ((u64)c0.w << 32);
      const u64 d2 = (u64)c1.z | ((u64)c1.w << 32);
      const u64 d3 = (u64)c2.x | ((u64)c2.y << 32);
      const u64 d4 = (u64)c2.z | ((u64)c2.w << 32);
      const u64 d5 = (u64)c3.x | ((u64)c3.y << 32);
      const u64 pa = (u64)c5.x | ((u64)c5.y << 32);
      const u64 pr = (u64)c5.z | ((u64)c5.w << 32);
      const double dl = ns_to_ms(d0), fwd = ns_to_ms(d2);
      const double bwd = ns_to_ms(d3), opt = ns_to_ms(d4), wall = ns_to_ms(d5);
      const bool has_mem = (rflags & TML_REC_HAS_MEM) != 0u;
      const bool usable = (dl > 0.0) || (fwd > 0.0) || (bwd > 0.0) || (opt > 0.0) || (wall > 0.0);
      const bool in_time = i >= t_start;
      const bool has_prev = i > 0, has_next = (i + 1) < n;
      const bool first_in_win = (i == t_start) || !has_prev || (prev_step != step);
      const bool last_m = !has_next || (next_step != step) || ((next_flags & TML_REC_HAS_MEM) == 0u);
      const bool cand_t = usable && in_time && first_in_win;
      const bool cand_m = has_mem && last_m;
      a_latest = step > a_latest ? step : a_latest;
      a_viol += (has_prev && step < prev_step) ? 1u : 0u;
      a_dups += (has_prev && step == prev_step) ? 1u : 0u;
      a_nr0 += in_time ? 1u : 0u;
      a_nr1 += has_mem ? 1u : 0u;
      if (cand_t) { a_lo0 = step < a_lo0 ? step : a_lo0; a_hi0 = step > a_hi0 ? step : a_hi0; ++a_nc0; }
      if (cand_m) { a_lo1 = step < a_lo1 ? step : a_lo1; a_hi1 = step > a_hi1 ? step : a_hi1; ++a_nc1; }
      a_both += (cand_t && cand_m) ? 1u : 0u;
      const double compute = (fwd + bwd) + opt;
      const double traced = fmax(wall, compute);      // model.py:246
      if (usable && in_time) {
        sums[0] += dl; sums[1] += fwd; sums[2] += bwd; sums[3] += opt;
        sums[4] += wall; sums[5] += traced; sums[6] += dl + traced;
        ++a_tc;
      }
      if (in_time) {
        a_sa += pa; a_sr += pr;
        mx_a = fmax(mx_a, (double)pa); mx_r = fmax(mx_r, (double)pr);
        // one rank: median == worst == the value (adapters.py:92-139 with a single column)
        const u64 j = i - t_start;
        const double wait = fmax(0.0, traced - compute);  // model.py:247
        const double va = (double)pa, vr = (double)pr;
        double* S = series + j;
        S[0 * n_ser] = dl;     S[1 * n_ser] = dl;
        S[2 * n_ser] = fwd;    S[3 * n_ser] = fwd;
        S[4 * n_ser] = bwd;    S[5 * n_ser] = bwd;
        S[6 * n_ser] = opt;    S[7 * n_ser] = opt;
        S[8 * n_ser] = traced; S[9 * n_ser] = traced;
        S[10 * n_ser] = wait;  S[11 * n_ser] = wait;
        S[12 * n_ser] = va;    S[13 * n_ser] = va;
        S[14 * n_ser] = vr;    S[15 * n_ser] = vr;
      }
    }
    __syncwarp();  // `cur` is free again
  }
  cp_async_wait<0>();
  {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      u64 t;
      t = __shfl_xor_sync(0xffffffffu, a_lo0, m); a_lo0 = t < a_lo0 ? t : a_lo0;
      t = __shfl_xor_sync(0xffffffffu, a_lo1, m); a_lo1 = t < a_lo1 ? t : a_lo1;
      t = __shfl_xor_sync(0xffffffffu, a_hi0, m); a_hi0 = t > a_hi0 ? t : a_hi0;
      t = __shfl_xor_sync(0xffffffffu, a_hi1, m); a_hi1 = t > a_hi1 ? t : a_hi1;
      t = __shfl_xor_sync(0xffffffffu, a_latest, m); a_latest = t > a_latest ? t : a_latest;
      a_sa += __shfl_xor_sync(0xffffffffu, a_sa, m); a_sr += __shfl_xor_sync(0xffffffffu, a_sr, m);
    }
    a_nc0 = __reduce_add_sync(0xffffffffu, a_nc0); a_nc1 = __reduce_add_sync(0xffffffffu, a_nc1);
    a_nr0 = __reduce_add_sync(0xffffffffu, a_nr0); a_nr1 = __reduce_add_sync(0xffffffffu, a_nr1);
    a_viol = __reduce_add_sync(0xffffffffu, a_viol); a_dups = __reduce_add_sync(0xffffffffu, a_dups);
    a_tc = __reduce_add_sync(0xffffffffu, a_tc); a_both = __reduce_add_sync(0xffffffffu, a_both);
    if (lane == 0) {
      if (a_nc0) { atomicMin(&acc->lo[0], a_lo0); atomicMax(&acc->hi[0], a_hi0); atomicAdd(&acc->ncand[0], (u64)a_nc0); }
      if (a_nc1) { atomicMin(&acc->lo[1], a_lo1); atomicMax(&acc->hi[1], a_hi1); atomicAdd(&acc->ncand[1], (u64)a_nc1); }
      if (a_nr0) atomicAdd(&acc->nrows[0], (u64)a_nr0);
      if (a_nr1) atomicAdd(&acc->nrows[1], (u64)a_nr1);
      atomicMax(&acc->latest_step, a_latest);
      if (a_viol) atomicAdd(&acc->violations, (u64)a_viol);
      if (a_dups) atomicAdd(&acc->dups, (u64)a_dups);
      if (a_tc) atomicAdd(&acc->t_count, (u64)a_tc);
      if (a_both) atomicAdd(&acc->n_both, (u64)a_both);
      if (a_sa) atomicAdd(&acc->msum[0], a_sa);
      if (a_sr) atomicAdd(&acc->msum[1], a_sr);
    }
  }
  __syncthreads();
  block_sum<9, WR_THREADS>(sums, partials + (size_t)blockIdx.x * 11);
  {
    __shared__ double s_mx[WR_THREADS / 32][2];
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      mx_a = fmax(mx_a, shfl_xor_f64(mx_a, m));
      mx_r = fmax(mx_r, shfl_xor_f64(mx_r, m));
    }
    if (lane == 0) { s_mx[warp][0] = mx_a; s_mx[warp][1] = mx_r; }
    __syncthreads();
    if (tid < 2) {
      double x = -INFINITY;
      for (int w = 0; w < WR_THREADS / 32; ++w) x = fmax(x, s_mx[w][tid]);
      partials[(size_t)blockIdx.x * 11 + 9 + tid] = x;
    }
  }
}

// ------------------------------------------------------------------ K3b: presence

__global__ void k_presence(const u64* __restrict__ steps, const u8* __restrict__ flags, u64 n,
                           u32 want, u64 glo, u64 span, u8* __restrict__ presence,
                           u32* __restrict__ rowof) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    if (flags[i] & want) {
      u64 s = steps[i];
      if (s >= glo && (s - glo) < span) {
        presence[s - glo] = 1;
        rowof[s - glo] = (u32)i;
      }
    }
  }
}

// ------------------------------------------------------------------ K3c: select
// exclusive scan of the presence bytes in three passes; keeps the last W ones.

#define SEL_THREADS 256
#define SEL_PER_THREAD 16
#define SEL_TILE (SEL_THREADS * SEL_PER_THREAD)

__device__ __forceinline__ u32 count16(const u8* __restrict__ p, u64 base, u64 span) {
  u32 c = 0;
  if (base + 16 <= span && ((base & 15ull) == 0ull)) {
    uint4 v = __ldg(reinterpret_cast<const uint4*>(p + base));
    // bytes are 0/1 -> popcount of the words counts the ones
    c = __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w);
  } else {
    for (int k = 0; k < 16; ++k) if (base + k < span) c += (p[base + k] != 0);
  }
  return c;
}

__global__ void __launch_bounds__(SEL_THREADS) k_sel_count(const u8* __restrict__ presence, u64 span,
                                                           u32* __restrict__ blockcnt) {
  __shared__ u32 s_w[SEL_THREADS / 32];
  u64 base = ((u64)blockIdx.x * SEL_THREADS + threadIdx.x) * SEL_PER_THREAD;
  u32 c = (base < span) ? count16(presence, base, span) : 0u;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    u32 t = 0;
    for (int w = 0; w < SEL_THREADS / 32; ++w) t += s_w[w];
    blockcnt[blockIdx.x] = t;
  }
}

// single block: exclusive scan of blockcnt[nb] in place, total -> *total_out
__global__ void __launch_bounds__(1024) k_sel_scan(u32* blockcnt, u32 nb, u64* total_out) {
  __shared__ u32 s_w[32];
  __shared__ u32 s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (u32 base = 0; base < nb; base += 1024) {
    u32 i = base + threadIdx.x;
    u32 v = (i < nb) ? blockcnt[i] : 0u;
    u32 incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      u32 t = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      u32 w = s_w[lane];
      u32 wi = w;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, wi, off);
        if (lane >= off) wi += t;
      }
      s_w[lane] = wi - w;  // exclusive warp offsets
    }
    __syncthreads();
    u32 carry = s_carry;
    u32 excl = carry + s_w[warp] + (incl - v);
    if (i < nb) blockcnt[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + s_w[warp] + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total_out = (u64)s_carry;
}

__global__ void __launch_bounds__(SEL_THREADS) k_sel_scatter(
    const u8* __restrict__ presence, u64 span, const u32* __restrict__ blockoff,
    const u64* __restrict__ total_p, u64 window, u64 glo, const u32* __restrict__ rowof,
    u32* __restrict__ sel_rows, u64* __restrict__ sel_steps) {
  __shared__ u32 s_w[SEL_THREADS / 32];
  const u64 total = *total_p;
  const u64 keep = total < window ? total : window;
  const u64 skip = total - keep;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u64 base = ((u64)blockIdx.x * SEL_THREADS + threadIdx.x) * SEL_PER_THREAD;
  u32 c = (base < span) ? count16(presence, base, span) : 0u;
  u32 incl = c;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    u32 t = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += t;
  }
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  u32 woff = 0;
  for (int w = 0; w < warp; ++w) woff += s_w[w];
  u64 rank = (u64)blockoff[blockIdx.x] + woff + (incl - c);
  if (c == 0u) return;
  for (int k = 0; k < SEL_PER_THREAD; ++k) {
    u64 i = base + k;
    if (i < span && presence[i]) {
      if (rank >= skip) {
        u64 j = rank - skip;
        sel_rows[j] = rowof[i];
        sel_steps[j] = glo + i;
      }
      ++rank;
    }
  }
}

// ------------------------------------------------------------------ K3d: gather
// thread = (row j, 16-B chunk q).  chunk roles: q0 (dl,h2d) q1 (fwd,bwd)
// q2 (opt,wall) q3 (alloc,resv).  Sums follow alignment.py:59-75.

#define GA_THREADS 256

// Are the selected rows one contiguous run of this rank's window rows?  (They are
// whenever the rank has no holes / duplicates inside the common window.)  Then the
// aligned rows ARE rows[first .. first+n) and k_gather skips the copy.
__global__ void k_check_contig(const u32* __restrict__ sel_rows, u64 nsel, u32* __restrict__ noncontig) {
  for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x + 1; j < nsel; j += (u64)gridDim.x * blockDim.x)
    if (sel_rows[j] != sel_rows[j - 1] + 1u) *noncontig = 1u;
}

__global__ void __launch_bounds__(GA_THREADS) k_gather(const tml_window_row* __restrict__ rows,
                                                      const u32* __restrict__ sel_rows, u64 nsel,
                                                      tml_window_row* __restrict__ xrows,
                                                      const u32* __restrict__ noncontig,
                                                      long long dense_first,
                                                      double* partials /* [grid][16] */,
                                                      u64* gacc /* [2]: exact byte sums (zeroed by the host) */) {
  __shared__ double s_part[GA_THREADS / 32][4][4];
  const uint4* rows4 = reinterpret_cast<const uint4*>(rows);
  uint4* x4 = reinterpret_cast<uint4*>(xrows);
  const int q = threadIdx.x & 3;
  const bool copy = (*noncontig) != 0u;
  double a0 = 0, a1 = 0, a2 = (q == 3) ? -INFINITY : 0.0, a3 = (q == 3) ? -INFINITY : 0.0;
  u64 ua = 0, ub = 0;  // q == 3: integer byte counts, summed exactly
  const u64 nthreads = (u64)gridDim.x * GA_THREADS;
  const u64 work = nsel * 4ull;
  // every thread of a 4-lane group runs the same trip count (work is a multiple of 4)
  // block-uniform trip count: the width-4 shuffles below need every lane of the warp
  for (u64 tb = (u64)blockIdx.x * GA_THREADS; tb < work; tb += nthreads) {
    const u64 t = tb + threadIdx.x;
    const bool ok = t < work;
    const u64 j = t >> 2;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (ok) {
      const u64 src = dense_first >= 0 ? (u64)dense_first + j : (u64)sel_rows[j];
      v = __ldg(&rows4[src * 4 + q]);
      if (copy) x4[j * 4 + q] = v;
    }
    double2 d = *reinterpret_cast<double2*>(&v);
    // q1 -> q2: fwd + bwd ; q0 -> q2: dl
    double fb = shfl_idx_f64(d.x + d.y, 1, 4);
    double dl = shfl_idx_f64(d.x, 0, 4);
    if (!ok) continue;
    if (q == 0) {
      a0 += d.x;
    } else if (q == 1) {
      a0 += d.x; a1 += d.y;
    } else if (q == 2) {
      const double compute = fb + d.x;         // (fwd + bwd) + opt
      const double traced = fmax(d.y, compute);
      a0 += d.x;                               // opt
      a1 += fmax(0.0, traced);                 // aligned step_cpu (alignment.py:72)
      a2 += traced;
      a3 += dl + traced;
    } else {
      ua += (u64)d.x; ub += (u64)d.y;  // integer-valued doubles < 2^53: the conversion is exact
      a2 = fmax(a2, d.x); a3 = fmax(a3, d.y);
    }
  }
  // reduce over lanes of the same chunk class (xor 4, 8, 16 keeps q)
  const bool is_max = (q == 3);
#pragma unroll
  for (int m = 4; m <= 16; m <<= 1) {
    a0 += shfl_xor_f64(a0, m);
    a1 += shfl_xor_f64(a1, m);
    double b2 = shfl_xor_f64(a2, m), b3 = shfl_xor_f64(a3, m);
    a2 = is_max ? fmax(a2, b2) : (a2 + b2);
    a3 = is_max ? fmax(a3, b3) : (a3 + b3);
    ua += __shfl_xor_sync(0xffffffffu, ua, m); ub += __shfl_xor_sync(0xffffffffu, ub, m);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 3 && gacc) {  // order-independent: integer atomics
    if (ua) atomicAdd(&gacc[0], ua);
    if (ub) atomicAdd(&gacc[1], ub);
  }
  if (lane < 4) {
    s_part[warp][lane][0] = a0; s_part[warp][lane][1] = a1;
    s_part[warp][lane][2] = a2; s_part[warp][lane][3] = a3;
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    const int qq = threadIdx.x >> 2, k = threadIdx.x & 3;
    const bool mx = (qq == 3) && (k >= 2);
    double x = mx ? -INFINITY : 0.0;
    for (int w = 0; w < GA_THREADS / 32; ++w) {
      double p = s_part[w][qq][k];
      x = mx ? fmax(x, p) : (x + p);
    }
    partials[(size_t)blockIdx.x * 16 + threadIdx.x] = x;
  }
}


// ------------------------------------------------------------------ K3e: reference-order sums
// Per-rank window means feed rank-level tie-breaks (closest-rank-to-median, argmax) that the
// reference decides on the last ulp, so the seven sums are reproduced in the reference's own
// order -- newest row first, one IEEE add after another (model.py:262-268, alignment.py:59-75)
// -- bit for bit.  Round 1 did that with one dependent DADD chain (10 ns/row, usable up to 2^17
// rows); tml_exact_sum.cuh does it for any window as composed integer maps.  A single-rank
// engine (world == 1) has nobody to break a tie against: above TML_EXACT_SUM_MAX rows it keeps
// the deterministic tree sums of K3a (rel <= 1e-13) and skips the two extra passes over its rows.

#define TML_EXACT_SUM_MAX (1u << 17)
#define XS_COMPOSE_CTAS_BESIDE_K4 0  // 0: no cap (smem allows 7 per SM)

#include "tml_exact_sum.cuh"

// ------------------------------------------------------------------ K4: window reduce

template <int R>
__device__ __forceinline__ void sort_small(double (&v)[R]) {
  // odd-even transposition network, fully unrolled: R values in registers
#pragma unroll
  for (int pass = 0; pass < R; ++pass) {
#pragma unroll
    for (int i = (pass & 1); i + 1 < R; i += 2) {
      double lo = fmin(v[i], v[i + 1]), hi = fmax(v[i], v[i + 1]);
      v[i] = lo; v[i + 1] = hi;
    }
  }
}

template <int R>
__device__ __forceinline__ void median_max(double (&v)[R], double& med, double& mx) {
  sort_small<R>(v);
  mx = v[R - 1];
  if (R & 1) med = v[R / 2];
  else med = (v[(R / 2 > 0 ? R / 2 : 1) - 1] + v[R / 2]) * 0.5;  // np.median / model.py:130-138
}

struct ReduceParams {
  const uint4* rows[TML_MAX_RANKS];
  double* series;
  u64 n_common, shard_lo, shard_hi;
  u32 mask;
  u32 n_ranks;
  unsigned long long* ticket;  // next tile to hand out (zeroed before the launch); NULL: static grid-stride
};

#define RD_THREADS 256

// Tile = 64 steps per CTA trip (256 threads = 64 steps x 4 chunks).  Results are staged
// in shared memory as [16 series][64 steps] and leave as 256-B contiguous warp stores
// (warp w writes series 2w and 2w+1), instead of sixteen 64-B fragments per warp: the
// kernel writes twice what it reads at small R, so store locality decides its HBM
// efficiency.
template <int R, int U>
__global__ void __launch_bounds__(RD_THREADS, (R <= 2 ? 8 : R <= 4 ? 5 : 3)) k_window_reduce(const __grid_constant__ ReduceParams p) {
  __shared__ double s_out[TML_SERIES_PER_STEP][RD_THREADS / 4];
  const int q = threadIdx.x & 3, row = threadIdx.x >> 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const u64 nthreads = (u64)gridDim.x * RD_THREADS;
  const u64 work = (p.shard_hi - p.shard_lo) * 4ull;
  const u64 n = p.n_common;
  double* __restrict__ S = p.series;
  const bool do_time = (p.mask & TML_MASK_TIME) != 0u, do_mem = (p.mask & TML_MASK_MEM) != 0u;
  // Tiles are handed out by a ticket counter, not by a fixed stride: beside K3e only part of the
  // grid is resident at first (the compose CTAs hold most of every SM for a while), and with a
  // fixed stride the CTAs that get in late would still have their whole share to do -- the kernel
  // would last until the last of them is done.  With tickets whoever is resident pulls work, late
  // CTAs find none.  Thread 0 draws the next ticket at the top of a trip (its latency hides under
  // the row loads) and publishes it between the trip's two barriers.
  __shared__ u64 s_tb;
  unsigned long long* const ticket = p.ticket;
  u64 tb = (u64)blockIdx.x * RD_THREADS;
  if (ticket) {
    if (threadIdx.x == 0) s_tb = (u64)atomicAdd(ticket, 1ull) * RD_THREADS;
    __syncthreads();
    tb = s_tb;
  }
  // block-uniform trip count: the width-4 shuffles and the barriers need every thread
  while (tb < work) {
    u64 next_tb = tb + nthreads;
    if (ticket && threadIdx.x == 0) next_tb = (u64)atomicAdd(ticket, 1ull) * RD_THREADS;
    const u64 t = tb + threadIdx.x;
    const bool ok = t < work;
    const u64 j = p.shard_lo + (t >> 2);
    double x[R], y[R], z[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {  // R independent 16-B loads in flight: local HBM or NVLink peer
      uint4 v = make_uint4(0, 0, 0, 0);
      if (ok) v = __ldg(&p.rows[r][j * 4 + q]);
      double2 d = *reinterpret_cast<double2*>(&v);
      x[r] = d.x; y[r] = d.y;
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      double fb = shfl_idx_f64(x[r] + y[r], 1, 4);   // fwd + bwd from q1
      if (q == 2) {
        const double compute = fb + x[r];            // (fwd + bwd) + opt
        const double traced = fmax(y[r], compute);   // model.py:246
        z[r] = fmax(0.0, traced - compute);          // model.py:247
        y[r] = traced;
      } else {
        z[r] = 0.0;
      }
    }
    double med, mx;
    if (q == 0) {
      median_max<R>(x, med, mx); s_out[0][row] = med; s_out[1][row] = mx;
    } else if (q == 1) {
      median_max<R>(x, med, mx); s_out[2][row] = med; s_out[3][row] = mx;
      median_max<R>(y, med, mx); s_out[4][row] = med; s_out[5][row] = mx;
    } else if (q == 2) {
      median_max<R>(x, med, mx); s_out[6][row] = med; s_out[7][row] = mx;
      median_max<R>(y, med, mx); s_out[8][row] = med; s_out[9][row] = mx;
      median_max<R>(z, med, mx); s_out[10][row] = med; s_out[11][row] = mx;
    } else {
      median_max<R>(x, med, mx); s_out[12][row] = med; s_out[13][row] = mx;
      median_max<R>(y, med, mx); s_out[14][row] = med; s_out[15][row] = mx;
    }
    __syncthreads();
    {
      const u64 tile_j = p.shard_lo + (tb >> 2);           // first step of this tile
      const u64 left = p.shard_hi - tile_j;                // steps of the tile that exist
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int sidx = warp * 2 + k;
        const bool on = sidx < 12 ? do_time : do_mem;
        if (on) {
          double* dst = S + (u64)sidx * n + tile_j;
          if ((u64)lane < left) dst[lane] = s_out[sidx][lane];
          if ((u64)lane + 32 < left) dst[lane + 32] = s_out[sidx][lane + 32];
        }
      }
    }
    if (ticket && threadIdx.x == 0) s_tb = next_tb;
    __syncthreads();
    tb = ticket ? s_tb : next_tb;
  }
}

// generic rank count (9..64): values in local memory, insertion sort
__global__ void __launch_bounds__(RD_THREADS) k_window_reduce_any(const __grid_constant__ ReduceParams p) {
  const int q = threadIdx.x & 3;
  const int R = (int)p.n_ranks;
  const u64 nthreads = (u64)gridDim.x * RD_THREADS;
  const u64 work = (p.shard_hi - p.shard_lo) * 4ull;
  const u64 n = p.n_common;
  double* __restrict__ S = p.series;
  const bool do_time = (p.mask & TML_MASK_TIME) != 0u, do_mem = (p.mask & TML_MASK_MEM) != 0u;
  for (u64 tb = (u64)blockIdx.x * RD_THREADS; tb < work; tb += nthreads) {
    const u64 t = tb + threadIdx.x;
    const bool ok = t < work;
    const u64 j = p.shard_lo + (t >> 2);
    double x[TML_MAX_RANKS], y[TML_MAX_RANKS], z[TML_MAX_RANKS];
    for (int r = 0; r < R; ++r) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (ok) v = __ldg(&p.rows[r][j * 4 + q]);
      double2 d = *reinterpret_cast<double2*>(&v);
      x[r] = d.x; y[r] = d.y;
      double fb = shfl_idx_f64(d.x + d.y, 1, 4);
      if (q == 2) {
        const double compute = fb + d.x;
        const double traced = fmax(d.y, compute);
        z[r] = fmax(0.0, traced - compute);
        y[r] = traced;
      } else {
        z[r] = 0.0;
      }
    }
    if (!ok) continue;
    auto mm = [&](double* v, double& med, double& mx) {
      for (int a = 1; a < R; ++a) {
        double key = v[a];
        int b = a - 1;
        while (b >= 0 && v[b] > key) { v[b + 1] = v[b]; --b; }
        v[b + 1] = key;
      }
      mx = v[R - 1];
      med = (R & 1) ? v[R / 2] : (v[R / 2 - 1] + v[R / 2]) * 0.5;
    };
    double med, mx;
    const bool tq = do_time && q < 3, mq = do_mem && q == 3;
    const int s0 = (q == 0) ? 0 : (q == 1) ? 2 : (q == 2) ? 6 : 12;
    if ((tq && q == 0)) { mm(x, med, mx); S[0 * n + j] = med; S[1 * n + j] = mx; }
    if ((tq && q >= 1) || mq) {
      mm(x, med, mx); S[(u64)s0 * n + j] = med; S[(u64)(s0 + 1) * n + j] = mx;
      mm(y, med, mx); S[(u64)(s0 + 2) * n + j] = med; S[(u64)(s0 + 3) * n + j] = mx;
    }
    if (tq && q == 2) { mm(z, med, mx); S[10 * n + j] = med; S[11 * n + j] = mx; }
  }
}

// ------------------------------------------------------------------ K4b: bands

struct BandParams {
  const double* series;
  u64 n_common, shard_lo, shard_hi;
  u64 lo[2][3], hi[2][3];
  u64 tail_first[2];
};

// grid (16 series, 4): y = 0..2 band sums over band ^ shard, y = 3 tail endpoints
__global__ void __launch_bounds__(256) k_bands(const __grid_constant__ BandParams p, double* out_sum,
                                               u64* out_cnt, double* out_tail) {
  const int s = blockIdx.x, b = blockIdx.y;
  const int kind = (s >= 12) ? 1 : 0;
  const double* v = p.series + (u64)s * p.n_common;
  if (b == 3) {
    if (threadIdx.x == 0) {
      u64 f = p.tail_first[kind], l = p.n_common ? p.n_common - 1 : 0;
      out_tail[s * 2 + 0] = (p.n_common && f >= p.shard_lo && f < p.shard_hi) ? v[f] : NAN;
      out_tail[s * 2 + 1] = (p.n_common && l >= p.shard_lo && l < p.shard_hi) ? v[l] : NAN;
    }
    return;
  }
  u64 lo = p.lo[kind][b], hi = p.hi[kind][b];
  if (lo < p.shard_lo) lo = p.shard_lo;
  if (hi > p.shard_hi) hi = p.shard_hi;
  double acc[1] = {0.0};
  for (u64 i = lo + threadIdx.x; i < hi; i += 256) acc[0] += v[i];
  double r[1];
  block_sum<1, 256>(acc, r);
  if (threadIdx.x == 0) {
    out_sum[s * 3 + b] = r[0];
    out_cnt[s * 3 + b] = (hi > lo) ? (hi - lo) : 0ull;
  }
}

// ------------------------------------------------------------------ K6: proc reduce
// columns: 0 sum_cpu 1 sum_rss 2 sum_used 3 sum_resv | max: 4 cpu 5 rss 6 used 7 resv
// 8 total 9 ratio 10 ts_max 11 -ts_min 12 cores 13 gpu_available | 14 n_gpu (sum)
// 15 sum_cpu low word: cpu% is the one non-integer column, and the reference's AVG is
// SQLite's compensated (Kahan-Babuska) sum, i.e. correctly rounded in practice.  The
// cpu sum is therefore carried as an unevaluated double-double (hi, lo) through every
// level of the reduction (TwoSum), so it rounds to the same double and rank-level
// tie-breaks on cpu_percent agree with the reference.

#define PR_THREADS 256
#define PR_COLS 16
#define PR_MAXMASK (((1u << 14) - 1u) & ~0xFu)

__device__ __forceinline__ void dd_add(double& hi, double& lo, double xh, double xl) {
  const double s = hi + xh;
  const double bp = s - hi;
  const double err = (hi - (s - bp)) + (xh - bp);
  hi = s;
  lo = (lo + xl) + err;
}

__global__ void __launch_bounds__(PR_THREADS) k_proc_reduce(const tml_proc_record* __restrict__ ring,
                                                           u32 slots, u64 first_k, u64 n,
                                                           double* partials) {
  __shared__ double s_part[PR_THREADS / 32][PR_COLS];
  double a[PR_COLS];
#pragma unroll
  for (int k = 0; k < PR_COLS; ++k) a[k] = ((PR_MAXMASK >> k) & 1u) ? -INFINITY : 0.0;
  for (u64 i = (u64)blockIdx.x * PR_THREADS + threadIdx.x; i < n; i += (u64)gridDim.x * PR_THREADS) {
    const uint4* p = reinterpret_cast<const uint4*>(&ring[(first_k + i) % slots]);
    uint4 c0 = __ldg(p), c1 = __ldg(p + 1), c2 = __ldg(p + 2), c3 = __ldg(p + 3);
    const double ts = __longlong_as_double((long long)((u64)c0.z | ((u64)c0.w << 32)));
    const double cpu = __longlong_as_double((long long)((u64)c1.x | ((u64)c1.y << 32)));
    const double rss = (double)((u64)c1.z | ((u64)c1.w << 32));
    const double used = (double)((u64)c2.x | ((u64)c2.y << 32));
    const double resv = (double)((u64)c2.z | ((u64)c2.w << 32));
    const double total = (double)((u64)c3.x | ((u64)c3.y << 32));
    const u32 fl = c3.z, cores = c3.w;
    dd_add(a[0], a[15], cpu, 0.0); a[4] = fmax(a[4], cpu);
    a[1] += rss; a[5] = fmax(a[5], rss);
    a[10] = fmax(a[10], ts); a[11] = fmax(a[11], -ts);
    a[12] = fmax(a[12], (double)cores);
    a[13] = fmax(a[13], (fl & TML_PROC_GPU_AVAILABLE) ? 1.0 : 0.0);
    if (fl & TML_PROC_HAS_GPU_METRICS) {
      a[2] += used; a[6] = fmax(a[6], used);
      a[3] += resv; a[7] = fmax(a[7], resv);
      a[8] = fmax(a[8], total);
      if (used > 0.0) a[9] = fmax(a[9], resv / used);  // loader.py:174-182
      a[14] += 1.0;
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {  // the double-double cpu sum
    const double oh = shfl_xor_f64(a[0], m), ol = shfl_xor_f64(a[15], m);
    dd_add(a[0], a[15], oh, ol);
  }
#pragma unroll
  for (int k = 1; k < PR_COLS - 1; ++k) {
    const bool mx = (PR_MAXMASK >> k) & 1u;
    double x = a[k];
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      double y = shfl_xor_f64(x, m);
      x = mx ? fmax(x, y) : (x + y);
    }
    a[k] = x;
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < PR_COLS; ++k) s_part[warp][k] = a[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double h = 0.0, l = 0.0;
    for (int w = 0; w < PR_THREADS / 32; ++w) dd_add(h, l, s_part[w][0], s_part[w][15]);
    partials[(size_t)blockIdx.x * PR_COLS + 0] = h;
    partials[(size_t)blockIdx.x * PR_COLS + 15] = l;
  } else if (threadIdx.x < PR_COLS - 1) {
    const bool mx = (PR_MAXMASK >> threadIdx.x) & 1u;
    double x = mx ? -INFINITY : 0.0;
    for (int w = 0; w < PR_THREADS / 32; ++w) {
      double y = s_part[w][threadIdx.x];
      x = mx ? fmax(x, y) : (x + y);
    }
    partials[(size_t)blockIdx.x * PR_COLS + threadIdx.x] = x;
  }
}

// fold the per-CTA (hi, lo) cpu sums with TwoSum -> out[hi_col], out[lo_col]: one warp,
// lane l folds CTAs l, l+32, ... then a shuffle tree of double-double adds (fixed order)
__global__ void k_finalize_dd(const double* __restrict__ partials, int nblk, int ncols, int hi_col,
                              int lo_col, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  double h = 0.0, l = 0.0;
  for (int b = lane; b < nblk; b += 32)
    dd_add(h, l, partials[(size_t)b * ncols + hi_col], partials[(size_t)b * ncols + lo_col]);
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const double oh = shfl_xor_f64(h, m), ol = shfl_xor_f64(l, m);
    dd_add(h, l, oh, ol);
  }
  if (lane == 0) { out[hi_col] = h; out[lo_col] = l; }
}

// =================================================================== host side

static thread_local char g_err[512] = "";

static int set_err(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

extern "C" int tml_set_error_(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define CK(call)                                                                         \
  do {                                                                                   \
    cudaError_t e_ = (call);                                                             \
    if (e_ != cudaSuccess)                                                               \
      return set_err(TML_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                     __FILE__, __LINE__);                                                \
  } while (0)

struct tml_ctx {
  int device = 0, rank = 0, world = 1;
  int n_sms = 132;
  u32 ring_slots = 0, proc_slots = 0, mirror_slots = 0, pmirror_slots = 0;
  DevState* d_state = nullptr;
  tml_step_record* d_ring = nullptr;
  tml_proc_record* d_pring = nullptr;
  HostPage* h_page = nullptr;        HostPage* d_page = nullptr;
  tml_step_record* h_mirror = nullptr; tml_step_record* d_mirror = nullptr;
  tml_proc_record* h_pmirror = nullptr; tml_proc_record* d_pmirror = nullptr;
  // host-side step state (training thread)
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;  // device time of k_window_rows alone
  cudaEvent_t ev2 = nullptr, ev3 = nullptr;  // device time of k_window_reduce alone
  unsigned long long* d_ticket = nullptr;    // K4's tile counter
  cudaEvent_t ev_proc = nullptr;             // the process aggregates have reached the staging slot
  u64 commits = 0;
  u64 launches = 0;  // kernels this context has launched (bench: gpu_launches)
  u32 next_slot = 0;
  u64 host_dur[TML_MAX_PHASES] = {0};
  u32 host_calls[TML_MAX_PHASES] = {0};
  // sampler-thread state
  std::atomic<u64> proc_commits{0};
  u64 drain_tail = 0, pdrain_tail = 0;
  u64 mirror_copied = 0;            // records k_mirror has brought to the host so far
  cudaStream_t drain_stream = nullptr;
  std::mutex mirror_mu;
  std::mutex proc_mu;
  // reduce workspace
  u64 cap_rows = 0;
  tml_window_row* d_rows = nullptr;
  u64* d_steps = nullptr;
  u8* d_flags = nullptr;
  u64 win_n = 0, win_tstart = 0;
  u64 win_ncand[2] = {0, 0};
  u64 win_lo[2] = {0, 0}, win_hi[2] = {0, 0};
  double win_tsums[7] = {0}, win_msums[4] = {0};  // sums over the whole time window (K3a)
  bool win_dense[2] = {false, false};
  bool win_ready = false;
  u64 cap_span[2] = {0, 0};
  u32* d_rowof[2] = {nullptr, nullptr};
  u64 cap_x[2] = {0, 0};
  tml_window_row* d_xrows[2] = {nullptr, nullptr};
  u64 n_common[2] = {0, 0};
  const tml_window_row* rows_ptr[2] = {nullptr, nullptr};  // aligned rows: d_xrows[k] or a slice of d_rows
  u32* d_noncontig = nullptr;
  u64 cap_sel = 0;
  u32* d_selrow = nullptr;
  u64* d_selstep = nullptr;
  u64 cap_blk = 0;
  u32* d_blockcnt = nullptr;
  u64* d_total = nullptr;
  WinAcc* d_winacc = nullptr;
  double* d_ppartials = nullptr; // proc reduce partials (own buffers: it overlaps the window reduce)
  double* d_pfinal = nullptr;
  bool proc_pending = false;
  u64 proc_pending_n = 0;
  u64* d_gacc = nullptr;         // k_gather's exact byte sums
  // K3e workspace (tml_exact_sum.cuh)
  u64 cap_xs = 0;                // chunks
  void* d_xs_buf = nullptr;      // one allocation, carved into XsWork
  XsWork xs_work;
  double* d_xs_out = nullptr; u64* d_xs_stats = nullptr;
  // deep profile (layer-id dimension)
  u32 n_layers = 0, layer_steps = 0, next_layer_slot = 0;
  LayerAcc* d_layer_acc = nullptr;
  tml_layer_record* d_layer_ring = nullptr;
  u64* d_layer_head = nullptr;
  u64 layer_commits = 0, layer_tail = 0;
  tml_layer_record* h_layer_stage = nullptr;  // pinned, one step's records
  cudaStream_t xs_stream = nullptr;  // K3e beside K4 (tml_win_set_defer)
  cudaEvent_t xs_gate = nullptr, xs_done = nullptr;
  bool xs_defer = false, xs_pending = false;
  double* d_partials = nullptr;  // max(grid) * 16 doubles
  double* d_final = nullptr;     // 64 doubles
  u64* d_bandcnt = nullptr;
  void* h_stage = nullptr;       // pinned 4 KB result staging
  std::unordered_map<std::string, void*> peers;
  void* comb[2] = {nullptr, nullptr};  // live step-combined workspaces, per kind (tml_combined.cuh)
  void* run_ws = nullptr;        // tml_reduce_run's workspace (tml_summary.cpp)
};

static void comb_free(tml_ctx* c);
extern "C" void** tml_run_ws_slot_(tml_ctx* c) { return &c->run_ws; }

static int grid_for(const tml_ctx* c, u64 work_items, int per_block) {
  u64 need = (work_items + per_block - 1) / per_block;
  u64 cap = (u64)c->n_sms * 4ull;  // persistent-style: a multiple of the SM count
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

// K3e workspace for `nchunks` chunks (one allocation, carved into XsWork)
static int xs_ensure(tml_ctx* c, long long nchunks) {
  if ((u64)nchunks <= c->cap_xs && c->d_xs_buf) return TML_OK;
  cudaFree(c->d_xs_buf);
  c->d_xs_buf = nullptr; c->cap_xs = 0;
  const u64 cap = (u64)nchunks + (u64)nchunks / 4 + 64, gcap = (cap + XS_GROUP - 1) / XS_GROUP + 1;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_csum = take(cap * 8 * sizeof(double)), o_cpre = take(cap * 8 * sizeof(double));
  const size_t nb_cap = (size_t)((cap + XS_WARPS - 1) / XS_WARPS + 1);
  const size_t o_btot = take(nb_cap * 8 * sizeof(double)), o_bpre = take(nb_cap * 8 * sizeof(double));
  const size_t o_plan = take(cap * 8 * sizeof(int)), o_ea = take(cap * 8 * sizeof(int));
  const size_t o_fn = take(cap * 7 * sizeof(XsFn)), o_gfn = take(gcap * 7 * sizeof(XsFn));
  const size_t o_gplan = take(gcap * 8 * sizeof(int)), o_tiles = take((size_t)XS_SLOT_CAP * sizeof(XsTileMaps));
  const size_t o_ns = take(256);
  CK(cudaMalloc(&c->d_xs_buf, off));
  char* base = (char*)c->d_xs_buf;
  XsWork w;
  w.csum = (double*)(base + o_csum); w.cpre = (double*)(base + o_cpre);
  w.btot = (double*)(base + o_btot); w.bpre = (double*)(base + o_bpre);
  w.plan = (int*)(base + o_plan); w.ea = (int*)(base + o_ea);
  w.fn = (XsFn*)(base + o_fn); w.gfn = (XsFn*)(base + o_gfn); w.gplan = (int*)(base + o_gplan);
  w.tiles = (XsTileMaps*)(base + o_tiles); w.nslots = (unsigned int*)(base + o_ns);
  c->xs_work = w;
  c->cap_xs = cap;
  return TML_OK;
}

// K3e launcher: the seven sums of `src` in reference order -> d_out[0..7) (device), on stream s.
// have_csum: the approximate chunk sums are already in the workspace (K3a put them there).
static int launch_exact_sums(tml_ctx* c, const XsSrc& src, double* d_out, cudaStream_t s, bool have_csum = false) {
  const long long n = src.last - src.first + 1 + src.pad;  // summation positions, leading pad included
  // one workspace per context: a job on another stream must wait for the deferred one
  if (c->xs_pending && s != c->xs_stream) CK(cudaStreamWaitEvent(s, c->xs_done, 0));
  if (n - src.pad <= 0) { CK(cudaMemsetAsync(d_out, 0, 7 * sizeof(double), s)); return TML_OK; }
  const long long nchunks = (n + XS_CHUNK - 1) / XS_CHUNK, ngroups = (nchunks + XS_GROUP - 1) / XS_GROUP;
  const int planned = n > 1024 ? 1 : 0;  // tiny windows: the walk adds / composes every tile itself
  const long long max_grid = (long long)c->n_sms * 8;
  {
    int rc = xs_ensure(c, nchunks);
    if (rc != TML_OK) return rc;
  }
  const XsWork& w = c->xs_work;
  if (planned) {
    const long long want = (nchunks + XS_WARPS - 1) / XS_WARPS;
    const int grid = (int)(want < max_grid ? want : max_grid);
    if (have_csum) k_xs_prefix<<<grid, 32, 0, s>>>(nchunks, w);
    else k_xs_partial<<<grid, XS_WARPS * 32, 0, s>>>(src, n, nchunks, w);
    CK(cudaPeekAtLastError());
    k_xs_bscan<<<1, 1024, 0, s>>>(w, grid);
    CK(cudaPeekAtLastError());
    {
      long long per = (nchunks + grid - 1) / grid;  // X1's run length (xs_block_range)
      per = (per + XS_WARPS - 1) / XS_WARPS * XS_WARPS;
      // beside K4 (deferred launch on the side stream) the compose CTAs must leave room for K4's:
      // dynamic shared memory that nobody touches caps them per SM (228 KB / (30 KB static + pad))
      static const int env_ctas = [] { const char* e = getenv("TML_XS_COMPOSE_CTAS"); return e ? atoi(e) : 0; }();
      int pad_bytes = 0;
      const int per_sm = env_ctas > 0 ? env_ctas : (s == c->xs_stream ? XS_COMPOSE_CTAS_BESIDE_K4 : 0);
      if (per_sm >= 1 && per_sm < 7) {
        pad_bytes = (int)(228 * 1024 / per_sm) - 32 * 1024;  // static 30 016 B + 1 KB reserved per CTA
        if (pad_bytes > 0) {
          static int attr_set = 0;
          if (attr_set < pad_bytes) {
            CK(cudaFuncSetAttribute(k_xs_compose, cudaFuncAttributeMaxDynamicSharedMemorySize, pad_bytes));
            attr_set = pad_bytes;
          }
        } else pad_bytes = 0;
      }
      k_xs_compose<<<(int)((nchunks + XS_CW - 1) / XS_CW), XS_CW * 32, pad_bytes, s>>>(src, n, nchunks, w, (int)per);
    }
    CK(cudaPeekAtLastError());
    k_xs_groups<<<(int)((ngroups * 7 + 7) / 8), 256, 0, s>>>(w, nchunks, ngroups);
    CK(cudaPeekAtLastError());
    c->launches += 4;
  }
  k_xs_walk<<<7, 256, 0, s>>>(src, n, nchunks, ngroups, w, planned, d_out, c->d_xs_stats);
  CK(cudaPeekAtLastError());
  c->launches += 1;
  return TML_OK;
}

static XsSrc xs_window_src(const tml_ctx* c, long long first, long long last) {
  XsSrc x;
  memset(&x, 0, sizeof(x));
  x.rows = c->d_rows; x.flags = c->d_flags; x.need = RF_USABLE | RF_IN_TIME;
  x.first = first; x.last = last; x.aligned = 0; x.dense_first = -1;
  x.pad = (XS_CHUNK - ((last + 1) % XS_CHUNK)) % XS_CHUNK;  // chunk boundaries on row indices: see XsSrc::pad
  return x;
}

extern "C" {

uint32_t tml_abi_version(void) { return TML_ABI_VERSION; }
const char* tml_last_error(void) { return g_err; }
const char* tml_status_str(int s) {
  switch (s) {
    case TML_OK: return "ok";
    case TML_ERR_CUDA: return "cuda error";
    case TML_ERR_ARG: return "bad argument";
    case TML_ERR_STATE: return "bad state";
    case TML_ERR_NOMEM: return "out of memory";
    case TML_ERR_NONMONOTONIC: return "step ids decrease inside the ring";
    case TML_ERR_UNSUPPORTED: return "unsupported";
    case TML_ERR_CAPTURE: return "stream is capturing";
    case TML_ERR_SMALL: return "buffer too small";
  }
  return "unknown";
}

int tml_init(int device, int rank, int world, uint32_t ring_slots, uint32_t proc_slots,
             tml_ctx** out) {
  if (!out || ring_slots == 0) return set_err(TML_ERR_ARG, "tml_init: bad arguments");
  if (proc_slots == 0) proc_slots = 1;
  CK(cudaSetDevice(device));
  tml_ctx* c = new (std::nothrow) tml_ctx();
  if (!c) return set_err(TML_ERR_NOMEM, "tml_init: host allocation failed");
  c->device = device; c->rank = rank; c->world = world;
  c->ring_slots = ring_slots; c->proc_slots = proc_slots;
  c->mirror_slots = ring_slots < 8192u ? ring_slots : 8192u;
  c->pmirror_slots = proc_slots < 16384u ? proc_slots : 16384u;
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  c->n_sms = sms > 0 ? sms : 132;
  CK(cudaMalloc(&c->d_state, sizeof(DevState)));
  CK(cudaMemset(c->d_state, 0, sizeof(DevState)));
  CK(cudaMalloc(&c->d_ring, (size_t)ring_slots * sizeof(tml_step_record)));
  CK(cudaMalloc(&c->d_pring, (size_t)proc_slots * sizeof(tml_proc_record)));
  CK(cudaHostAlloc(&c->h_page, sizeof(HostPage), cudaHostAllocMapped));
  memset(c->h_page, 0, sizeof(HostPage));
  CK(cudaHostGetDevicePointer((void**)&c->d_page, c->h_page, 0));
  CK(cudaHostAlloc(&c->h_mirror, (size_t)c->mirror_slots * sizeof(tml_step_record), cudaHostAllocMapped));
  CK(cudaHostGetDevicePointer((void**)&c->d_mirror, c->h_mirror, 0));
  CK(cudaHostAlloc(&c->h_pmirror, (size_t)c->pmirror_slots * sizeof(tml_proc_record), cudaHostAllocMapped));
  CK(cudaHostGetDevicePointer((void**)&c->d_pmirror, c->h_pmirror, 0));
  CK(cudaMalloc(&c->d_total, sizeof(u64)));
  CK(cudaMalloc(&c->d_noncontig, sizeof(u32)));
  CK(cudaMalloc(&c->d_gacc, 2 * sizeof(u64)));
  CK(cudaMalloc(&c->d_xs_out, 16 * sizeof(double)));
  CK(cudaMalloc(&c->d_xs_stats, 8 * sizeof(u64)));
  CK(cudaMalloc(&c->d_partials, (size_t)c->n_sms * 4 * 16 * sizeof(double)));
  CK(cudaMalloc(&c->d_final, 64 * sizeof(double) + sizeof(WinAcc)));
  c->d_winacc = reinterpret_cast<WinAcc*>(c->d_final + 64);  // one D2H copy fetches both
  CK(cudaMalloc(&c->d_ppartials, (size_t)c->n_sms * 4 * 16 * sizeof(double)));
  CK(cudaMalloc(&c->d_pfinal, 32 * sizeof(double)));
  CK(cudaMalloc(&c->d_bandcnt, 64 * sizeof(u64)));
  CK(cudaHostAlloc(&c->h_stage, 4096, cudaHostAllocDefault));
  *out = c;
  return TML_OK;
}

int tml_shutdown(tml_ctx* c) {
  if (!c) return TML_OK;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (auto& kv : c->peers) cudaIpcCloseMemHandle(kv.second);
  cudaFree(c->d_state); cudaFree(c->d_ring); cudaFree(c->d_pring);
  cudaFreeHost(c->h_page); cudaFreeHost(c->h_mirror); cudaFreeHost(c->h_pmirror);
  cudaFree(c->d_rows); cudaFree(c->d_steps); cudaFree(c->d_flags);
  for (int k = 0; k < 2; ++k) { cudaFree(c->d_rowof[k]); cudaFree(c->d_xrows[k]); }
  cudaFree(c->d_selrow); cudaFree(c->d_selstep); cudaFree(c->d_blockcnt); cudaFree(c->d_total);
  cudaFree(c->d_noncontig); cudaFree(c->d_gacc);
  cudaFree(c->d_xs_buf); cudaFree(c->d_xs_out); cudaFree(c->d_xs_stats);
  cudaFree(c->d_layer_acc); cudaFree(c->d_layer_ring); cudaFree(c->d_layer_head);
  if (c->h_layer_stage) cudaFreeHost(c->h_layer_stage);
  if (c->drain_stream) cudaStreamDestroy(c->drain_stream);
  if (c->xs_stream) cudaStreamDestroy(c->xs_stream);
  if (c->xs_gate) cudaEventDestroy(c->xs_gate);
  if (c->xs_done) cudaEventDestroy(c->xs_done);
  if (c->d_ticket) cudaFree(c->d_ticket);
  cudaFree(c->d_partials); cudaFree(c->d_final); cudaFree(c->d_bandcnt);
  cudaFree(c->d_ppartials); cudaFree(c->d_pfinal);
  cudaFreeHost(c->h_stage);
  comb_free(c);
  tml_run_ws_free_(c->run_ws);
  delete c;
  return TML_OK;
}

// ---------------------------------------------------------------- step path

// Entry points may be called from any host thread (a fresh thread's current device is 0): make the
// context's device current before launching on one of its streams.  cudaGetDevice is a TLS read.
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(const tml_ctx* c) {
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != c->device) { prev = cur; cudaSetDevice(c->device); }
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }  // the caller's current device is restored
};

static inline int check_capture(cudaStream_t s) {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &st) != cudaSuccess) { cudaGetLastError(); return 0; }
  return st != cudaStreamCaptureStatusNone;
}

int tml_phase_begin(tml_ctx* c, uint32_t phase, void* stream) {
  if (!c || phase >= TML_MAX_PHASES) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  if (check_capture(s)) return TML_ERR_CAPTURE;
  u32 slot = c->next_slot;
  c->next_slot = (slot + 1u) % TML_N_SLOTS;
  k_stamp_begin<<<1, 32, 0, s>>>(c->d_state, slot);
  c->launches += 1;
  if (cudaPeekAtLastError() != cudaSuccess)
    return set_err(TML_ERR_CUDA, "stamp_begin launch: %s", cudaGetErrorString(cudaGetLastError()));
  return (int)slot;
}

int tml_phase_end(tml_ctx* c, uint32_t phase, int slot, void* stream) {
  if (!c || phase >= TML_MAX_PHASES || slot < 0 || slot >= (int)TML_N_SLOTS) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  if (check_capture(s)) return TML_ERR_CAPTURE;
  k_stamp_end<<<1, 32, 0, s>>>(c->d_state, (u32)slot, phase, (u32)(c->commits % TML_N_EPOCHS));
  c->launches += 1;
  if (cudaPeekAtLastError() != cudaSuccess)
    return set_err(TML_ERR_CUDA, "stamp_end launch: %s", cudaGetErrorString(cudaGetLastError()));
  return TML_OK;
}

// ---------------------------------------------------------------- deep profile
int tml_layer_init(tml_ctx* c, uint32_t n_layers, uint32_t steps) {
  if (!c || n_layers == 0 || steps == 0) return TML_ERR_ARG;
  DeviceGuard dg(c);
  cudaFree(c->d_layer_acc); cudaFree(c->d_layer_ring); cudaFree(c->d_layer_head);
  if (c->h_layer_stage) cudaFreeHost(c->h_layer_stage);
  c->d_layer_acc = nullptr; c->d_layer_ring = nullptr; c->d_layer_head = nullptr; c->h_layer_stage = nullptr;
  CK(cudaMalloc(&c->d_layer_acc, (size_t)n_layers * sizeof(LayerAcc)));
  CK(cudaMemset(c->d_layer_acc, 0, (size_t)n_layers * sizeof(LayerAcc)));
  CK(cudaMalloc(&c->d_layer_ring, (size_t)n_layers * steps * sizeof(tml_layer_record)));
  CK(cudaMalloc(&c->d_layer_head, sizeof(u64)));
  CK(cudaMemset(c->d_layer_head, 0, sizeof(u64)));
  CK(cudaHostAlloc(&c->h_layer_stage, ((size_t)n_layers * sizeof(tml_layer_record)) + 64, cudaHostAllocDefault));
  c->n_layers = n_layers; c->layer_steps = steps; c->layer_commits = 0; c->layer_tail = 0;
  return TML_OK;
}

int tml_layer_begin(tml_ctx* c, void* stream) {
  if (!c || !c->n_layers) return TML_ERR_STATE;
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  if (check_capture(s)) return TML_ERR_CAPTURE;
  const u32 slot = c->next_layer_slot;
  c->next_layer_slot = (slot + 1u) % TML_N_SLOTS;
  k_layer_begin<<<1, 32, 0, s>>>(c->d_state, slot);
  c->launches += 1;
  if (cudaPeekAtLastError() != cudaSuccess)
    return set_err(TML_ERR_CUDA, "layer_begin launch: %s", cudaGetErrorString(cudaGetLastError()));
  return (int)slot;
}

int tml_layer_end(tml_ctx* c, uint32_t layer, uint32_t direction, int slot, uint64_t bytes, void* stream) {
  if (!c || !c->n_layers || layer >= c->n_layers || direction > 1 || slot < 0 || slot >= (int)TML_N_SLOTS)
    return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  if (check_capture(s)) return TML_ERR_CAPTURE;
  k_layer_end<<<1, 32, 0, s>>>(c->d_state, c->d_layer_acc, (u32)slot, layer, direction, bytes);
  c->launches += 1;
  if (cudaPeekAtLastError() != cudaSuccess)
    return set_err(TML_ERR_CUDA, "layer_end launch: %s", cudaGetErrorString(cudaGetLastError()));
  return TML_OK;
}

int tml_layer_commit(tml_ctx* c, uint64_t step, void* stream) {
  if (!c || !c->n_layers) return TML_ERR_STATE;
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  if (check_capture(s)) return TML_ERR_CAPTURE;
  const int blocks = (int)((c->n_layers + 255) / 256);
  k_layer_commit<<<blocks, 256, 0, s>>>(c->d_layer_acc, c->d_layer_ring, c->n_layers, c->layer_steps,
                                        c->layer_commits, step, c->d_layer_head);
  if (blocks > 1) k_layer_head<<<1, 1, 0, s>>>(c->d_layer_head, c->layer_commits + 1);
  CK(cudaPeekAtLastError());
  c->launches += blocks > 1 ? 2 : 1;
  c->layer_commits += 1;
  return TML_OK;
}

int tml_layer_drain(tml_ctx* c, tml_layer_record* out, uint32_t max_steps, uint32_t* n_steps, uint32_t* n_layers,
                    uint64_t* n_dropped) {
  if (!c || !out || !n_steps) return TML_ERR_ARG;
  *n_steps = 0;
  if (n_layers) *n_layers = c->n_layers;
  if (n_dropped) *n_dropped = 0;
  if (!c->n_layers) return TML_OK;
  DeviceGuard dg(c);
  std::lock_guard<std::mutex> g(c->mirror_mu);
  if (!c->drain_stream) CK(cudaStreamCreateWithFlags(&c->drain_stream, cudaStreamNonBlocking));
  u64 head = 0;
  CK(cudaMemcpyAsync(c->h_layer_stage, c->d_layer_head, sizeof(u64), cudaMemcpyDeviceToHost, c->drain_stream));
  CK(cudaStreamSynchronize(c->drain_stream));
  memcpy(&head, c->h_layer_stage, sizeof(u64));
  u64 tail = c->layer_tail;
  if (head - tail > c->layer_steps) { if (n_dropped) *n_dropped = head - tail - c->layer_steps; tail = head - c->layer_steps; }
  u32 n = 0;
  const size_t row = (size_t)c->n_layers * sizeof(tml_layer_record);
  while (tail < head && n < max_steps) {
    CK(cudaMemcpyAsync(out + (size_t)n * c->n_layers, c->d_layer_ring + (size_t)(tail % c->layer_steps) * c->n_layers,
                       row, cudaMemcpyDeviceToHost, c->drain_stream));
    ++n; ++tail;
  }
  CK(cudaStreamSynchronize(c->drain_stream));
  c->layer_tail = tail;
  *n_steps = n;
  return TML_OK;
}

int tml_phase_host(tml_ctx* c, uint32_t phase, uint64_t dur_ns) {
  if (!c || phase >= TML_MAX_PHASES) return TML_ERR_ARG;
  c->host_dur[phase] += dur_ns;
  c->host_calls[phase] += 1u;
  return TML_OK;
}

int tml_step_discard(tml_ctx* c) {
  if (!c) return TML_ERR_ARG;
  memset(c->host_dur, 0, sizeof(c->host_dur));
  memset(c->host_calls, 0, sizeof(c->host_calls));
  return TML_OK;
}

int tml_step_commit(tml_ctx* c, uint64_t step, uint64_t peak_alloc, uint64_t peak_resv,
                    uint32_t flags, double host_ts, void* stream) {
  if (!c) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  if (check_capture(s)) return TML_ERR_CAPTURE;
  CommitArgs a;
  a.step = step; a.host_ts = host_ts;
  memcpy(a.host_dur, c->host_dur, sizeof(a.host_dur));
  memcpy(a.host_calls, c->host_calls, sizeof(a.host_calls));
  a.epoch = (u32)(c->commits % TML_N_EPOCHS);
  a.flags = flags;
  a.peak_alloc = peak_alloc;
  a.peak_resv = peak_resv;
  a.seq = c->commits;
  k_commit<<<1, 192, 0, s>>>(c->d_state, c->d_ring, c->ring_slots, a);
  memset(c->host_dur, 0, sizeof(c->host_dur));
  memset(c->host_calls, 0, sizeof(c->host_calls));
  if (cudaPeekAtLastError() != cudaSuccess)
    return set_err(TML_ERR_CUDA, "commit launch: %s", cudaGetErrorString(cudaGetLastError()));
  c->commits += 1;
  c->launches += 1;
  c->win_ready = false;
  return TML_OK;
}

uint64_t tml_step_count(tml_ctx* c) { return c ? c->commits : 0; }
uint64_t tml_launch_count(tml_ctx* c) { return c ? c->launches : 0; }
uint64_t tml_proc_count(tml_ctx* c) { return c ? c->proc_commits.load() : 0; }

// ---------------------------------------------------------------- sampler side

// bring the host mirror up to date (sampler thread, own stream; never the training stream)
static int refresh_mirror(tml_ctx* c) {
  DeviceGuard dg(c);
  std::lock_guard<std::mutex> g(c->mirror_mu);
  if (!c->drain_stream) CK(cudaStreamCreateWithFlags(&c->drain_stream, cudaStreamNonBlocking));
  k_mirror<<<1, 1024, 0, c->drain_stream>>>(c->d_state, c->d_ring, c->ring_slots, c->d_mirror, c->mirror_slots,
                                            c->d_page, c->mirror_copied);
  CK(cudaPeekAtLastError());
  CK(cudaStreamSynchronize(c->drain_stream));
  c->mirror_copied = c->h_page->mirror_head;
  return TML_OK;
}

int tml_drain(tml_ctx* c, tml_step_record* out, uint32_t max_records, uint32_t* n_out,
              uint64_t* n_dropped) {
  if (!c || !out || !n_out) return TML_ERR_ARG;
  if (c->drain_tail >= c->h_page->mirror_head) {  // nothing left over from the last refresh
    int rc = refresh_mirror(c);
    if (rc != TML_OK) return rc;
  }
  u64 head = c->h_page->mirror_head;
  std::atomic_thread_fence(std::memory_order_acquire);
  u64 tail = c->drain_tail, dropped = 0;
  if (head - tail > c->mirror_slots) { dropped = head - tail - c->mirror_slots; tail = head - c->mirror_slots; }
  u32 n = 0;
  while (tail < head && n < max_records) {
    memcpy(&out[n], (const void*)&c->h_mirror[tail % c->mirror_slots], sizeof(tml_step_record));
    ++n; ++tail;
  }
  c->drain_tail = tail;
  *n_out = n;
  if (n_dropped) *n_dropped = dropped;
  return TML_OK;
}

int tml_proc_drain(tml_ctx* c, tml_proc_record* out, uint32_t max_records, uint32_t* n_out,
                   uint64_t* n_dropped) {
  if (!c || !out || !n_out) return TML_ERR_ARG;
  u64 head = c->h_page->pmirror_head;
  std::atomic_thread_fence(std::memory_order_acquire);
  u64 tail = c->pdrain_tail, dropped = 0;
  if (head - tail > c->pmirror_slots) { dropped = head - tail - c->pmirror_slots; tail = head - c->pmirror_slots; }
  u32 n = 0;
  while (tail < head && n < max_records) {
    memcpy(&out[n], (const void*)&c->h_pmirror[tail % c->pmirror_slots], sizeof(tml_proc_record));
    ++n; ++tail;
  }
  c->pdrain_tail = tail;
  *n_out = n;
  if (n_dropped) *n_dropped = dropped;
  return TML_OK;
}

int tml_live(tml_ctx* c, tml_live_stats* out) {
  if (!c || !out) return TML_ERR_ARG;
  {
    int rc = refresh_mirror(c);
    if (rc != TML_OK) return rc;
  }
  memcpy(out, (const void*)&c->h_page->live, sizeof(tml_live_stats));
  return TML_OK;
}

int tml_proc_commit(tml_ctx* c, const tml_proc_record* sample, void* stream) {
  if (!c || !sample) return TML_ERR_ARG;
  std::lock_guard<std::mutex> g(c->proc_mu);
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);  // the sampler thread is not the training thread
  k_proc_commit<<<1, 32, 0, s>>>(c->d_state, c->d_pring, c->proc_slots, c->d_pmirror,
                                  c->pmirror_slots, c->d_page, *sample);
  c->launches += 1;
  if (cudaPeekAtLastError() != cudaSuccess)
    return set_err(TML_ERR_CUDA, "proc_commit launch: %s", cudaGetErrorString(cudaGetLastError()));
  c->proc_commits.fetch_add(1);
  return TML_OK;
}

static int load_span(void* d_ring, u32 slots, size_t rec_bytes, u64 start, const void* host, u64 n,
                     cudaStream_t s) {
  // at most two contiguous spans (ring wrap); if n > slots only the last `slots` survive
  const char* src = (const char*)host;
  if (n > slots) { src += (size_t)(n - slots) * rec_bytes; start += (n - slots); n = slots; }
  u64 pos = start % slots;
  u64 first = (pos + n <= slots) ? n : (slots - pos);
  CK(cudaMemcpyAsync((char*)d_ring + pos * rec_bytes, src, (size_t)first * rec_bytes,
                     cudaMemcpyHostToDevice, s));
  if (first < n)
    CK(cudaMemcpyAsync(d_ring, src + (size_t)first * rec_bytes, (size_t)(n - first) * rec_bytes,
                       cudaMemcpyHostToDevice, s));
  return TML_OK;
}

__global__ void k_set_heads(DevState* st, u64 head, u64 proc_head, int which) {
  if (which == 0) st->head = head; else st->proc_head = proc_head;
}

int tml_ring_load(tml_ctx* c, const tml_step_record* host, uint64_t n, void* stream) {
  if (!c || (!host && n)) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  int rc = load_span(c->d_ring, c->ring_slots, sizeof(tml_step_record), c->commits, host, n, s);
  if (rc != TML_OK) return rc;
  c->commits += n;
  k_set_heads<<<1, 1, 0, s>>>(c->d_state, c->commits, 0, 0);
  CK(cudaPeekAtLastError());
  c->win_ready = false;
  // bulk-loaded history is not new telemetry: the sampler's cursor starts behind it
  c->mirror_copied = c->drain_tail = c->commits;
  c->h_page->mirror_head = c->commits;
  return TML_OK;
}

int tml_proc_load(tml_ctx* c, const tml_proc_record* host, uint64_t n, void* stream) {
  if (!c || (!host && n)) return TML_ERR_ARG;
  std::lock_guard<std::mutex> g(c->proc_mu);
  cudaStream_t s = (cudaStream_t)stream;
  u64 cur = c->proc_commits.load();
  int rc = load_span(c->d_pring, c->proc_slots, sizeof(tml_proc_record), cur, host, n, s);
  if (rc != TML_OK) return rc;
  c->proc_commits.store(cur + n);
  k_set_heads<<<1, 1, 0, s>>>(c->d_state, 0, cur + n, 1);
  CK(cudaPeekAtLastError());
  return TML_OK;
}

int tml_ring_reset(tml_ctx* c) {
  if (!c) return TML_ERR_ARG;
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemset(c->d_state, 0, sizeof(DevState)));
  memset(c->h_page, 0, sizeof(HostPage));
  c->commits = 0; c->proc_commits.store(0); c->next_slot = 0;
  c->drain_tail = 0; c->pdrain_tail = 0; c->mirror_copied = 0;
  memset(c->host_dur, 0, sizeof(c->host_dur));
  memset(c->host_calls, 0, sizeof(c->host_calls));
  c->win_ready = false;
  return TML_OK;
}

// ---------------------------------------------------------------- reduce

}  // extern "C"

template <typename T>
static int ensure(T** p, u64* cap, u64 need, bool exact_alloc = false) {
  if (need <= *cap && *p) return TML_OK;
  if (*p) { cudaFree(*p); *p = nullptr; *cap = 0; }
  u64 n = need < 1 ? 1 : need;
  if (!exact_alloc) n = n + n / 4 + 64;
  cudaError_t e = cudaMalloc((void**)p, (size_t)n * sizeof(T));
  if (e != cudaSuccess) return set_err(TML_ERR_NOMEM, "cudaMalloc(%llu B): %s",
                                       (u64)(n * sizeof(T)), cudaGetErrorString(e));
  *cap = n;
  return TML_OK;
}

extern "C" {

int tml_win_prepare(tml_ctx* c, uint32_t window, void* stream, tml_win_info* out) {
  if (!c || !out || window == 0) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  memset(out, 0, sizeof(*out));
  const u64 n = c->commits < c->ring_slots ? c->commits : c->ring_slots;
  const u64 first_k = c->commits - n;
  c->win_n = n;
  c->win_tstart = n > window ? n - window : 0;
  out->n_retained = n;
  out->monotone = 1;
  c->win_ncand[0] = c->win_ncand[1] = 0;
  if (c->xs_pending) {  // the previous reduce's K3e still reads the rows this call rewrites
    CK(cudaStreamWaitEvent(s, c->xs_done, 0));
    c->xs_pending = false;
  }
  if (n == 0) {
    memset(c->win_tsums, 0, sizeof(c->win_tsums));
    memset(c->win_msums, 0, sizeof(c->win_msums));
    c->win_ready = true;
    return TML_OK;
  }
  int rc;
  u64 cap = c->cap_rows;
  if (n > cap) {
    cudaFree(c->d_rows); cudaFree(c->d_steps); cudaFree(c->d_flags);
    c->d_rows = nullptr; c->d_steps = nullptr; c->d_flags = nullptr; c->cap_rows = 0;
    u64 want = n + n / 4 + 64;
    if (want > c->ring_slots) want = c->ring_slots;
    if (want < n) want = n;
    CK(cudaMalloc(&c->d_rows, (size_t)want * sizeof(tml_window_row)));
    CK(cudaMalloc(&c->d_steps, (size_t)want * sizeof(u64)));
    CK(cudaMalloc(&c->d_flags, (size_t)want));
    c->cap_rows = want;
  }
  WinAcc init;
  memset(&init, 0, sizeof(init));
  init.lo[0] = init.lo[1] = ~0ull;
  CK(cudaMemcpyAsync(c->d_winacc, &init, sizeof(init), cudaMemcpyHostToDevice, s));
  static bool wr_attr = false;
  if (!wr_attr) {
    CK(cudaFuncSetAttribute(k_window_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, WR_SMEM_BYTES));
    wr_attr = true;
  }
  int grid = (int)((n + WR_THREADS - 1) / WR_THREADS);
  if (grid > c->n_sms * 2) grid = c->n_sms * 2;  // 2 resident CTAs per SM (83 KB smem each)
  if (!c->ev0) { CK(cudaEventCreate(&c->ev0)); CK(cudaEventCreate(&c->ev1)); }
  // K3e (reference-order sums) needs approximate 256-row chunk sums for its plan: K3a has every row
  // in registers anyway and adds them up on the way (tml_exact_sum.cuh: X1 without a pass of its own)
  bool exact_win = c->world > 1 || (n - c->win_tstart) <= TML_EXACT_SUM_MAX;
  const XsSrc wsrc = xs_window_src(c, (long long)c->win_tstart, (long long)n - 1);
  const long long w_pos = (long long)(n - c->win_tstart) + wsrc.pad;
  static const bool env_csum = [] { const char* e = getenv("TML_XS_K3A_CSUM"); return !e || e[0] != '0'; }();
  const bool k3a_csum = exact_win && w_pos > 1024 && env_csum;
  double* d_csum = nullptr;
  if (k3a_csum) {
    if (c->xs_pending) { CK(cudaStreamWaitEvent(s, c->xs_done, 0)); c->xs_pending = false; }
    const long long nchunks = (w_pos + XS_CHUNK - 1) / XS_CHUNK;
    int xr = xs_ensure(c, nchunks);
    if (xr != TML_OK) return xr;
    d_csum = c->xs_work.csum;
    CK(cudaMemsetAsync(d_csum, 0, (size_t)nchunks * 8 * sizeof(double), s));
  }
  CK(cudaEventRecord(c->ev0, s));
  k_window_rows<<<grid, WR_THREADS, WR_SMEM_BYTES, s>>>(c->d_ring, c->ring_slots, first_k, n, c->win_tstart,
                                            c->d_rows, c->d_steps, c->d_flags, c->d_winacc,
                                            c->d_partials, d_csum, (u64)(n - 1 + wsrc.pad));
  CK(cudaPeekAtLastError());
  CK(cudaEventRecord(c->ev1, s));
  k_finalize<<<1, 32 * 11, 0, s>>>(c->d_partials, grid, 11, (1u << 9) | (1u << 10), c->d_final + 32);
  CK(cudaPeekAtLastError());
  c->launches += 2;  // K3a + its finalize
  if (exact_win && c->xs_defer) {
    // beside the row exchange / K4: side stream, gated on K3a; the tree sums stand in until
    // tml_win_exact_collect
    if (!c->xs_stream) {
      int prio_lo = 0, prio_hi = 0;  // highest priority: K3e's CTAs are placed before K4's when slots free up
      CK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
      CK(cudaStreamCreateWithPriority(&c->xs_stream, cudaStreamNonBlocking, prio_hi));
      CK(cudaEventCreateWithFlags(&c->xs_gate, cudaEventDisableTiming));
      CK(cudaEventCreate(&c->xs_done));  // timed: tml_kernel_ms(3)
    }
    CK(cudaEventRecord(c->xs_gate, s));
    CK(cudaStreamWaitEvent(c->xs_stream, c->xs_gate, 0));
    int xr = launch_exact_sums(c, wsrc, c->d_xs_out, c->xs_stream, k3a_csum);
    if (xr != TML_OK) return xr;
    CK(cudaEventRecord(c->xs_done, c->xs_stream));
    c->xs_pending = true;
    exact_win = false;
  } else if (exact_win) {  // reference-order sums (used instead of the tree sums)
    int xr = launch_exact_sums(c, wsrc, c->d_final, s, k3a_csum);
    if (xr != TML_OK) return xr;
  }
  // d_final[0..7) exact sums | d_final[32..43) tree sums + maxima | d_final[64..] WinAcc: one copy
  char* st = (char*)c->h_stage;
  CK(cudaMemcpyAsync(st + 1024, c->d_final, 64 * sizeof(double) + sizeof(WinAcc), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  memcpy(st, st + 1024 + 64 * sizeof(double), sizeof(WinAcc));
  memcpy(st + 256, st + 1024 + (exact_win ? 0 : 32) * sizeof(double), 7 * sizeof(double));
  memcpy(st + 320, st + 1024 + (32 + 7) * sizeof(double), 4 * sizeof(double));
  WinAcc acc;
  memcpy(&acc, st, sizeof(acc));
  memcpy(out->t_sums, st + 256, 7 * sizeof(double));
  memcpy(c->win_msums, st + 320, 4 * sizeof(double));
  c->win_msums[0] = (double)acc.msum[0];  // exact integer sums, rounded once (u64 -> f64 is RN)
  c->win_msums[1] = (double)acc.msum[1];
  memcpy(c->win_tsums, out->t_sums, 7 * sizeof(double));
  out->latest_step = acc.latest_step;
  out->monotone = acc.violations == 0 ? 1u : 0u;
  out->dup_rows = (u32)acc.dups;
  for (int k = 0; k < 2; ++k) {
    out->n_rows[k] = acc.nrows[k];
    out->n_cand[k] = acc.ncand[k];
    out->lo[k] = acc.ncand[k] ? acc.lo[k] : 0;
    out->hi[k] = acc.ncand[k] ? acc.hi[k] : 0;
  }
  out->t_count = acc.t_count;
  out->n_both = acc.n_both;
  {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev0, c->ev1) == cudaSuccess) out->kernel_ms = (double)ms;
  }
  c->win_ncand[0] = acc.ncand[0]; c->win_ncand[1] = acc.ncand[1];
  // dense: every window row is a candidate and the candidates' step ids are consecutive, so
  // row(step) = first_row + (step - lo) and the aligned rows are a contiguous slice
  const u64 rows_in[2] = {n - c->win_tstart, n};
  for (int k = 0; k < 2; ++k) {
    c->win_lo[k] = out->lo[k]; c->win_hi[k] = out->hi[k];
    c->win_dense[k] = acc.ncand[k] > 0 && acc.ncand[k] == rows_in[k] &&
                      (out->hi[k] - out->lo[k] + 1) == acc.ncand[k];
    out->dense[k] = c->win_dense[k] ? 1u : 0u;
  }
  c->win_ready = true;
  (void)rc;
  if (!out->monotone)
    return set_err(TML_ERR_NONMONOTONIC, "step ids decrease inside the retained ring (%llu places)",
                   acc.violations);
  return TML_OK;
}

int tml_win_peek(tml_ctx* c, uint32_t window, uint64_t* n_retained, uint64_t* n_window) {
  if (!c || window == 0) return TML_ERR_ARG;
  const u64 n = c->commits < c->ring_slots ? c->commits : c->ring_slots;
  if (n_retained) *n_retained = n;
  if (n_window) *n_window = n > window ? window : n;
  return TML_OK;
}

// Single-rank bulk path: ring -> per-step series in ONE pass (k_window_fused).  *ok = 1: the
// window is dense and `series` ([16][n_window], device) plus `aligned` hold the result; 0: the
// caller runs the staged path (tml_win_prepare ...).  Leaves no WindowRows behind.
int tml_win_fused(tml_ctx* c, uint32_t window, double* series, void* stream, tml_win_info* out,
                  tml_align_info* aligned, uint32_t* ok) {
  if (!c || !out || !aligned || !ok || !series || window == 0) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  memset(out, 0, sizeof(*out));
  memset(aligned, 0, sizeof(*aligned));
  *ok = 0;
  const u64 n = c->commits < c->ring_slots ? c->commits : c->ring_slots;
  const u64 first_k = c->commits - n;
  const u64 t_start = n > window ? n - window : 0;
  const u64 n_win = n - t_start;
  c->win_ready = false;
  out->n_retained = n;
  out->monotone = 1;
  if (n == 0) return TML_OK;
  if (c->xs_pending) { CK(cudaStreamWaitEvent(s, c->xs_done, 0)); c->xs_pending = false; }
  WinAcc init;
  memset(&init, 0, sizeof(init));
  init.lo[0] = init.lo[1] = ~0ull;
  CK(cudaMemcpyAsync(c->d_winacc, &init, sizeof(init), cudaMemcpyHostToDevice, s));
  static bool wf_attr = false;
  if (!wf_attr) {
    CK(cudaFuncSetAttribute(k_window_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, WF_SMEM_BYTES));
    wf_attr = true;
  }
  int grid = (int)((n + WR_THREADS - 1) / WR_THREADS);
  if (grid > c->n_sms * 2) grid = c->n_sms * 2;
  if (!c->ev0) { CK(cudaEventCreate(&c->ev0)); CK(cudaEventCreate(&c->ev1)); }
  CK(cudaEventRecord(c->ev0, s));
  k_window_fused<<<grid, WR_THREADS, WF_SMEM_BYTES, s>>>(c->d_ring, c->ring_slots, first_k, n, t_start, series, n_win,
                                                          c->d_winacc, c->d_partials);
  CK(cudaPeekAtLastError());
  CK(cudaEventRecord(c->ev1, s));
  k_finalize<<<1, 32 * 11, 0, s>>>(c->d_partials, grid, 11, (1u << 9) | (1u << 10), c->d_final + 32);
  CK(cudaPeekAtLastError());
  c->launches += 2;
  char* st = (char*)c->h_stage;
  CK(cudaMemcpyAsync(st + 1024, c->d_final, 64 * sizeof(double) + sizeof(WinAcc), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  WinAcc acc;
  memcpy(&acc, st + 1024 + 64 * sizeof(double), sizeof(acc));
  double f[11];
  memcpy(f, st + 1024 + 32 * sizeof(double), sizeof(f));
  memcpy(out->t_sums, f, 7 * sizeof(double));
  out->latest_step = acc.latest_step;
  out->monotone = acc.violations == 0 ? 1u : 0u;
  out->dup_rows = (u32)acc.dups;
  const u64 rows_in[2] = {n_win, n};
  for (int k = 0; k < 2; ++k) {
    out->n_rows[k] = acc.nrows[k];
    out->n_cand[k] = acc.ncand[k];
    out->lo[k] = acc.ncand[k] ? acc.lo[k] : 0;
    out->hi[k] = acc.ncand[k] ? acc.hi[k] : 0;
    out->dense[k] = (acc.ncand[k] > 0 && acc.ncand[k] == rows_in[k] &&
                     (out->hi[k] - out->lo[k] + 1) == acc.ncand[k]) ? 1u : 0u;
  }
  out->t_count = acc.t_count;
  out->n_both = acc.n_both;
  {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev0, c->ev1) == cudaSuccess) out->kernel_ms = (double)ms;
  }
  if (!out->monotone)
    return set_err(TML_ERR_NONMONOTONIC, "step ids decrease inside the retained ring (%llu places)", acc.violations);
  // dense in both kinds: the last min(n, W) memory candidates are exactly the time window's rows
  if (out->dense[0] && out->dense[1] && out->hi[0] == out->hi[1] && acc.ncand[0] == n_win) {
    *ok = 1;
    aligned->n_common = n_win;
    aligned->start_step = out->lo[0];
    aligned->end_step = out->hi[0];
    aligned->n_rows = n_win;
    memcpy(aligned->t_sums, out->t_sums, 7 * sizeof(double));
    aligned->t_sums[4] = out->t_sums[5];  // aligned step_cpu = sum of traced (alignment.py:72)
    aligned->m_sums[0] = (double)acc.msum[0]; aligned->m_sums[1] = (double)acc.msum[1];
    aligned->m_sums[2] = f[9]; aligned->m_sums[3] = f[10];
  }
  return TML_OK;
}

int tml_win_set_defer(tml_ctx* c, int on) {
  if (!c) return TML_ERR_ARG;
  c->xs_defer = on != 0;
  return TML_OK;
}

int tml_win_exact_collect(tml_ctx* c, void* stream, double t_sums[7]) {
  if (!c || !t_sums) return TML_ERR_ARG;
  if (!c->win_ready) return set_err(TML_ERR_STATE, "tml_win_exact_collect before tml_win_prepare");
  if (c->xs_pending) {
    cudaStream_t s = (cudaStream_t)stream;
    CK(cudaSetDevice(c->device));
    CK(cudaStreamWaitEvent(s, c->xs_done, 0));
    char* st = (char*)c->h_stage;
    CK(cudaMemcpyAsync(st + 448, c->d_xs_out, 7 * sizeof(double), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    memcpy(c->win_tsums, st + 448, 7 * sizeof(double));
    c->xs_pending = false;
  }
  memcpy(t_sums, c->win_tsums, 7 * sizeof(double));
  return TML_OK;
}

int tml_win_exact_stats(tml_ctx* c, uint64_t slow_rows[7]) {
  if (!c || !slow_rows) return TML_ERR_ARG;
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpy(slow_rows, c->d_xs_stats, 7 * sizeof(u64), cudaMemcpyDeviceToHost));
  return TML_OK;
}

int tml_win_presence(tml_ctx* c, uint32_t kind, uint64_t glo, uint64_t span, uint8_t* presence,
                     void* stream) {
  if (!c || kind > 1 || !presence || span == 0) return TML_ERR_ARG;
  if (!c->win_ready) return set_err(TML_ERR_STATE, "tml_win_presence before tml_win_prepare");
  if (span >> 32) return set_err(TML_ERR_UNSUPPORTED, "step-id span %llu too wide", (u64)span);
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  int rc = ensure(&c->d_rowof[kind], &c->cap_span[kind], span);
  if (rc != TML_OK) return rc;
  // a rank without candidates must not constrain the intersection: all ones
  if (c->win_n == 0 || c->win_ncand[kind] == 0) { CK(cudaMemsetAsync(presence, 1, span, s)); return TML_OK; }
  CK(cudaMemsetAsync(presence, 0, span, s));
  const u32 want = kind == TML_KIND_TIME ? RF_CAND_T : RF_CAND_M;
  const int grid = grid_for(c, c->win_n, 256);
  k_presence<<<grid, 256, 0, s>>>(c->d_steps, c->d_flags, c->win_n, want, glo, span, presence,
                                  c->d_rowof[kind]);
  CK(cudaPeekAtLastError());
  c->launches += 1;
  return TML_OK;
}

int tml_win_select(tml_ctx* c, uint32_t kind, uint64_t glo, uint64_t span, const uint8_t* presence,
                   uint32_t window, void* stream, tml_align_info* out) {
  if (!c || kind > 1 || !out || window == 0) return TML_ERR_ARG;
  if (!c->win_ready) return set_err(TML_ERR_STATE, "tml_win_select before tml_win_prepare");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  memset(out, 0, sizeof(*out));
  c->n_common[kind] = 0;
  c->rows_ptr[kind] = nullptr;
  if (span == 0 || !presence) return TML_OK;
  const u32 nb = (u32)((span + SEL_TILE - 1) / SEL_TILE);
  int rc = ensure(&c->d_blockcnt, &c->cap_blk, nb);
  if (rc != TML_OK) return rc;
  const u64 maxsel = span < window ? span : window;
  if (maxsel > c->cap_sel) {
    cudaFree(c->d_selrow); cudaFree(c->d_selstep);
    c->d_selrow = nullptr; c->d_selstep = nullptr; c->cap_sel = 0;
    CK(cudaMalloc(&c->d_selrow, (size_t)maxsel * sizeof(u32)));
    CK(cudaMalloc(&c->d_selstep, (size_t)maxsel * sizeof(u64)));
    c->cap_sel = maxsel;
  }
  rc = ensure(&c->d_xrows[kind], &c->cap_x[kind], maxsel, true);
  if (rc != TML_OK) return rc;
  k_sel_count<<<nb, SEL_THREADS, 0, s>>>(presence, span, c->d_blockcnt);
  CK(cudaPeekAtLastError());
  k_sel_scan<<<1, 1024, 0, s>>>(c->d_blockcnt, nb, c->d_total);
  CK(cudaPeekAtLastError());
  k_sel_scatter<<<nb, SEL_THREADS, 0, s>>>(presence, span, c->d_blockcnt, c->d_total, (u64)window,
                                           glo, c->d_rowof[kind], c->d_selrow, c->d_selstep);
  CK(cudaPeekAtLastError());
  c->launches += 3;
  char* st = (char*)c->h_stage;
  CK(cudaMemcpyAsync(st, c->d_total, sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  u64 total = 0;
  memcpy(&total, st, sizeof(u64));
  const u64 keep = total < window ? total : window;
  c->n_common[kind] = keep;
  out->n_common = keep;
  if (keep == 0) return TML_OK;
  // a rank that has no candidates of its own does not own rows for the window
  if (c->win_n == 0 || c->win_ncand[kind] == 0) return TML_OK;
  const int grid = grid_for(c, keep * 4, GA_THREADS);
  CK(cudaMemsetAsync(c->d_noncontig, 0, sizeof(u32), s));
  k_check_contig<<<grid_for(c, keep, 256), 256, 0, s>>>(c->d_selrow, keep, c->d_noncontig);
  CK(cudaPeekAtLastError());
  CK(cudaMemsetAsync(c->d_gacc, 0, 2 * sizeof(u64), s));
  k_gather<<<grid, GA_THREADS, 0, s>>>(c->d_rows, c->d_selrow, keep, c->d_xrows[kind], c->d_noncontig,
                                       -1ll, c->d_partials, c->d_gacc);
  CK(cudaPeekAtLastError());
  c->launches += 1;
  k_finalize<<<1, 32 * 16, 0, s>>>(c->d_partials, grid, 16, (1u << 14) | (1u << 15), c->d_final);
  CK(cudaPeekAtLastError());
  c->launches += 2;
  const bool exact = (kind == TML_KIND_TIME) && (c->world > 1 || keep <= TML_EXACT_SUM_MAX);
  if (exact) {
    XsSrc x;
    memset(&x, 0, sizeof(x));
    x.rows = c->d_rows; x.first = 0; x.last = (long long)keep - 1; x.aligned = 1;
    x.xrows = c->d_xrows[kind]; x.noncontig = c->d_noncontig; x.sel_rows = c->d_selrow; x.dense_first = -1;
    int xr = launch_exact_sums(c, x, c->d_final + 16, s);
    if (xr != TML_OK) return xr;
    CK(cudaMemcpyAsync(st + 320, c->d_final + 16, 7 * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaMemcpyAsync(st + 400, c->d_gacc, 2 * sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 64, c->d_final, 16 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 256, c->d_selstep, sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 264, c->d_selstep + (keep - 1), sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 272, c->d_noncontig, sizeof(u32), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 276, c->d_selrow, sizeof(u32), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  {
    u32 noncontig = 0, first_row = 0;
    memcpy(&noncontig, st + 272, sizeof(u32));
    memcpy(&first_row, st + 276, sizeof(u32));
    c->rows_ptr[kind] = noncontig ? c->d_xrows[kind] : (c->d_rows + first_row);
  }
  double f[16];
  memcpy(f, st + 64, sizeof(f));
  // partial layout [q][k]: q0 {dl} q1 {fwd,bwd} q2 {opt,cpu,traced,total} q3 {alloc,resv,maxa,maxr}
  out->t_sums[0] = f[0]; out->t_sums[1] = f[4]; out->t_sums[2] = f[5]; out->t_sums[3] = f[8];
  out->t_sums[4] = f[9]; out->t_sums[5] = f[10]; out->t_sums[6] = f[11];
  out->m_sums[0] = f[12]; out->m_sums[1] = f[13]; out->m_sums[2] = f[14]; out->m_sums[3] = f[15];
  {
    u64 g[2];
    memcpy(g, st + 400, sizeof(g));
    out->m_sums[0] = (double)g[0]; out->m_sums[1] = (double)g[1];  // exact integer sums, rounded once
  }
  if (exact) memcpy(out->t_sums, st + 320, 7 * sizeof(double));
  memcpy(&out->start_step, st + 256, sizeof(u64));
  memcpy(&out->end_step, st + 264, sizeof(u64));
  out->n_rows = keep;
  return TML_OK;
}

int tml_win_select_dense(tml_ctx* c, uint32_t kind, uint64_t first_step, uint64_t n_common,
                         void* stream, tml_align_info* out) {
  if (!c || kind > 1 || !out) return TML_ERR_ARG;
  if (!c->win_ready) return set_err(TML_ERR_STATE, "tml_win_select_dense before tml_win_prepare");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  memset(out, 0, sizeof(*out));
  c->n_common[kind] = n_common;
  c->rows_ptr[kind] = nullptr;
  out->n_common = n_common;
  if (n_common == 0 || c->win_n == 0 || c->win_ncand[kind] == 0) return TML_OK;
  if (!c->win_dense[kind] || first_step < c->win_lo[kind] ||
      first_step + n_common - 1 > c->win_hi[kind])
    return set_err(TML_ERR_STATE, "window is not dense over the requested steps");
  const u64 first_row = (kind == TML_KIND_TIME ? c->win_tstart : 0) + (first_step - c->win_lo[kind]);
  c->rows_ptr[kind] = c->d_rows + first_row;
  if (kind == TML_KIND_TIME && first_step == c->win_lo[kind] && n_common == c->win_ncand[kind]) {
    // the common window IS this rank's whole time window (ranks in lock step): the sums
    // k_window_rows already produced are the aligned sums -- nothing left to launch.
    // (aligned step_cpu = sum of traced: alignment.py:72 -> t_sums[4] := t_sums[5])
    memcpy(out->t_sums, c->win_tsums, sizeof(c->win_tsums));
    out->t_sums[4] = c->win_tsums[5];
    memcpy(out->m_sums, c->win_msums, sizeof(c->win_msums));
    out->start_step = first_step;
    out->end_step = first_step + n_common - 1;
    out->n_rows = n_common;
    return TML_OK;
  }
  const int grid = grid_for(c, n_common * 4, GA_THREADS);
  CK(cudaMemsetAsync(c->d_noncontig, 0, sizeof(u32), s));
  CK(cudaMemsetAsync(c->d_gacc, 0, 2 * sizeof(u64), s));
  k_gather<<<grid, GA_THREADS, 0, s>>>(c->d_rows, nullptr, n_common, nullptr, c->d_noncontig,
                                       (long long)first_row, c->d_partials, c->d_gacc);
  CK(cudaPeekAtLastError());
  k_finalize<<<1, 32 * 16, 0, s>>>(c->d_partials, grid, 16, (1u << 14) | (1u << 15), c->d_final);
  CK(cudaPeekAtLastError());
  c->launches += 2;
  const bool exact = (kind == TML_KIND_TIME) && (c->world > 1 || n_common <= TML_EXACT_SUM_MAX);
  char* st = (char*)c->h_stage;
  if (exact) {
    XsSrc x;
    memset(&x, 0, sizeof(x));
    x.rows = c->d_rows; x.first = 0; x.last = (long long)n_common - 1; x.aligned = 1;
    x.dense_first = (long long)first_row;
    int xr = launch_exact_sums(c, x, c->d_final + 16, s);
    if (xr != TML_OK) return xr;
    CK(cudaMemcpyAsync(st + 320, c->d_final + 16, 7 * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaMemcpyAsync(st + 400, c->d_gacc, 2 * sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 64, c->d_final, 16 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  double f[16];
  memcpy(f, st + 64, sizeof(f));
  out->t_sums[0] = f[0]; out->t_sums[1] = f[4]; out->t_sums[2] = f[5]; out->t_sums[3] = f[8];
  out->t_sums[4] = f[9]; out->t_sums[5] = f[10]; out->t_sums[6] = f[11];
  out->m_sums[0] = f[12]; out->m_sums[1] = f[13]; out->m_sums[2] = f[14]; out->m_sums[3] = f[15];
  {
    u64 g[2];
    memcpy(g, st + 400, sizeof(g));
    out->m_sums[0] = (double)g[0]; out->m_sums[1] = (double)g[1];  // exact integer sums, rounded once
  }
  if (exact) memcpy(out->t_sums, st + 320, 7 * sizeof(double));
  out->start_step = first_step;
  out->end_step = first_step + n_common - 1;
  out->n_rows = n_common;
  return TML_OK;
}

const void* tml_win_rows(tml_ctx* c, uint32_t kind) {
  if (!c || kind > 1) return nullptr;
  return c->rows_ptr[kind];
}

int tml_win_rows_export(tml_ctx* c, uint32_t kind, void* handle64, uint64_t* byte_offset) {
  if (!c || kind > 1 || !handle64 || !byte_offset) return TML_ERR_ARG;
  if (!c->rows_ptr[kind]) return set_err(TML_ERR_STATE, "no aligned rows to export");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle is 64 B");
  CK(cudaSetDevice(c->device));
  // IPC handles name whole allocations: export the base and the slice's offset
  const char* p = (const char*)c->rows_ptr[kind];
  const char* base = (p >= (const char*)c->d_rows && p < (const char*)(c->d_rows + c->cap_rows))
                         ? (const char*)c->d_rows : (const char*)c->d_xrows[kind];
  CK(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)handle64, (void*)base));
  *byte_offset = (uint64_t)(p - base);
  return TML_OK;
}

int tml_peer_open(tml_ctx* c, const void* handle64, void** peer_ptr) {
  if (!c || !handle64 || !peer_ptr) return TML_ERR_ARG;
  CK(cudaSetDevice(c->device));
  std::string key((const char*)handle64, 64);
  auto it = c->peers.find(key);
  if (it != c->peers.end()) { *peer_ptr = it->second; return TML_OK; }
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  c->peers.emplace(key, p);
  *peer_ptr = p;
  return TML_OK;
}

int tml_peer_close(tml_ctx* c, void* peer_ptr) {
  if (!c || !peer_ptr) return TML_ERR_ARG;
  for (auto it = c->peers.begin(); it != c->peers.end(); ++it) {
    if (it->second == peer_ptr) {
      CK(cudaIpcCloseMemHandle(peer_ptr));
      c->peers.erase(it);
      return TML_OK;
    }
  }
  return TML_ERR_ARG;
}

}  // extern "C"

template <int R>
static void launch_reduce(int grid, cudaStream_t s, const ReduceParams& p) {
  constexpr int U = 1;  // one row in flight per thread; occupancy hides the latency
  k_window_reduce<R, U><<<grid, RD_THREADS, 0, s>>>(p);
}

extern "C" {

int tml_win_reduce(tml_ctx* c, const tml_reduce_args* a, void* stream) {
  if (!c || !a || !a->series || a->n_ranks == 0 || a->n_ranks > TML_MAX_RANKS) return TML_ERR_ARG;
  if (a->shard_hi > a->n_common || a->shard_lo > a->shard_hi) return TML_ERR_ARG;
  if (a->shard_hi == a->shard_lo) return TML_OK;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  ReduceParams p;
  memset(&p, 0, sizeof(p));
  for (u32 r = 0; r < a->n_ranks; ++r) {
    if (!a->rows[r]) return set_err(TML_ERR_ARG, "rows[%u] is NULL", r);
    p.rows[r] = (const uint4*)a->rows[r];
  }
  p.series = a->series; p.n_common = a->n_common;
  p.shard_lo = a->shard_lo; p.shard_hi = a->shard_hi;
  p.mask = a->mask; p.n_ranks = a->n_ranks;
  // A multiple of the SM count; the CTAs pull tiles from a ticket counter.  One rank: 8 CTAs/SM
  // (29 regs), HBM-bound.  Several ranks: NVLink-bound -- two CTAs of 256 threads x R loads already
  // keep several bandwidth-delay products in flight per SM -- and K3e runs beside it on the side
  // stream, so the cap leaves the registers of one walk CTA free on every SM (without it the
  // persistent K4 CTAs hold every SM and the walk starts only when K4 has finished).
  u64 need = ((a->shard_hi - a->shard_lo) * 4 + RD_THREADS - 1) / RD_THREADS;
  static const int env_ctas = [] { const char* e = getenv("TML_K4_CTAS"); return e ? atoi(e) : 0; }();
  // registers decide what fits beside K3e's walk (16 K): R = 2: 6 x 8 K, R = 3..4: 4 x 12 K, R >= 5: 2 x 20 K
  // (re-measured on the H100: DESIGN.md, "Launch shapes on the H100")
  const u64 per_sm = env_ctas > 0 ? (u64)env_ctas
                     : (a->n_ranks >= 5 ? 2ull : a->n_ranks >= 3 ? 4ull : a->n_ranks > 1 ? 6ull : 8ull);
  const u64 cap = (u64)c->n_sms * per_sm;
  const int grid = (int)(need < cap ? (need ? need : 1) : cap);
  if (!c->ev2) { CK(cudaEventCreate(&c->ev2)); CK(cudaEventCreate(&c->ev3)); }
  static const bool env_ticket = [] { const char* e = getenv("TML_K4_TICKET"); return !e || e[0] != '0'; }();
  if (env_ticket && a->n_ranks <= 8) {
    if (!c->d_ticket) CK(cudaMalloc(&c->d_ticket, sizeof(unsigned long long)));
    CK(cudaMemsetAsync(c->d_ticket, 0, sizeof(unsigned long long), s));
    p.ticket = c->d_ticket;
  }
  CK(cudaEventRecord(c->ev2, s));
  switch (a->n_ranks) {
    case 1: launch_reduce<1>(grid, s, p); break;
    case 2: launch_reduce<2>(grid, s, p); break;
    case 3: launch_reduce<3>(grid, s, p); break;
    case 4: launch_reduce<4>(grid, s, p); break;
    case 5: launch_reduce<5>(grid, s, p); break;
    case 6: launch_reduce<6>(grid, s, p); break;
    case 7: launch_reduce<7>(grid, s, p); break;
    case 8: launch_reduce<8>(grid, s, p); break;
    default: k_window_reduce_any<<<grid, RD_THREADS, 0, s>>>(p); break;
  }
  CK(cudaPeekAtLastError());
  CK(cudaEventRecord(c->ev3, s));
  c->launches += 1;
  return TML_OK;
}

double tml_kernel_ms(tml_ctx* c, uint32_t which) {
  if (!c || which > 4) return -1.0;
  cudaEvent_t a = which == 1 ? c->ev2 : c->ev0;
  cudaEvent_t b = which == 0 ? c->ev1 : which == 2 ? c->ev2 : which == 3 ? c->xs_done : c->ev3;
  if (!a || !b) return -1.0;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, a, b) != cudaSuccess) { cudaGetLastError(); return -1.0; }
  return (double)ms;
}

int tml_win_bands(tml_ctx* c, const double* series, const tml_band_args* a, void* stream,
                  tml_band_out* out) {
  if (!c || !series || !a || !out) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  BandParams p;
  p.series = series; p.n_common = a->n_common; p.shard_lo = a->shard_lo; p.shard_hi = a->shard_hi;
  memcpy(p.lo, a->band_lo, sizeof(p.lo));
  memcpy(p.hi, a->band_hi, sizeof(p.hi));
  memcpy(p.tail_first, a->tail_first, sizeof(p.tail_first));
  double* d_sum = c->d_final;            // 48 doubles
  double* d_tail = c->d_partials;        // 32 doubles (scratch)
  k_bands<<<dim3(16, 4), 256, 0, s>>>(p, d_sum, c->d_bandcnt, d_tail);
  CK(cudaPeekAtLastError());
  c->launches += 1;
  char* st = (char*)c->h_stage;
  CK(cudaMemcpyAsync(st, d_sum, 48 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 512, c->d_bandcnt, 48 * sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 1024, d_tail, 32 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  memcpy(out->sum, st, 48 * sizeof(double));
  memcpy(out->cnt, st + 512, 48 * sizeof(u64));
  double tails[32];
  memcpy(tails, st + 1024, sizeof(tails));
  for (int k = 0; k < 16; ++k) { out->tail_first[k] = tails[2 * k]; out->tail_last[k] = tails[2 * k + 1]; }
  return TML_OK;
}

// Launch half: kernels + the async copy of the 16 result doubles into a private
// staging slot.  The result is complete after ANY later synchronisation of `stream`
// (tml_win_prepare synchronises it), so the reduce pays no separate sync for it.
int tml_proc_reduce_launch(tml_ctx* c, uint32_t max_rows, void* stream) {
  if (!c || max_rows == 0) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  const u64 total = c->proc_commits.load();
  u64 n = total < c->proc_slots ? total : c->proc_slots;
  if (n > max_rows) n = max_rows;
  c->proc_pending_n = n;
  c->proc_pending = true;
  if (n == 0) return TML_OK;
  const u64 first_k = total - n;
  const int grid = grid_for(c, n, PR_THREADS);
  k_proc_reduce<<<grid, PR_THREADS, 0, s>>>(c->d_pring, c->proc_slots, first_k, n, c->d_ppartials);
  CK(cudaPeekAtLastError());
  k_finalize<<<1, 32 * PR_COLS, 0, s>>>(c->d_ppartials, grid, PR_COLS, PR_MAXMASK, c->d_pfinal);
  CK(cudaPeekAtLastError());
  k_finalize_dd<<<1, 32, 0, s>>>(c->d_ppartials, grid, PR_COLS, 0, 15, c->d_pfinal);
  CK(cudaPeekAtLastError());
  c->launches += 3;
  CK(cudaMemcpyAsync((char*)c->h_stage + 3072, c->d_pfinal, PR_COLS * sizeof(double),
                     cudaMemcpyDeviceToHost, s));
  if (!c->ev_proc) CK(cudaEventCreateWithFlags(&c->ev_proc, cudaEventDisableTiming));
  CK(cudaEventRecord(c->ev_proc, s));
  return TML_OK;
}

int tml_proc_reduce_collect(tml_ctx* c, tml_proc_agg* out) {
  if (!c || !out) return TML_ERR_ARG;
  if (!c->proc_pending) return set_err(TML_ERR_STATE, "tml_proc_reduce_collect without a launch");
  c->proc_pending = false;
  memset(out, 0, sizeof(*out));
  out->max_ratio = -1.0;
  const u64 n = c->proc_pending_n;
  if (n == 0) return TML_OK;
  // normally complete already (tml_win_prepare synchronised the stream); an empty step
  // ring returns from there without a sync, so wait on the copy itself
  CK(cudaEventSynchronize(c->ev_proc));
  double f[PR_COLS];
  memcpy(f, (char*)c->h_stage + 3072, sizeof(f));
  out->n = n;
  out->n_gpu = (u64)f[14];
  out->sum_cpu = f[0]; out->sum_cpu_lo = f[15]; out->max_cpu = f[4];
  out->sum_rss = f[1]; out->max_rss = f[5];
  out->sum_used = f[2]; out->max_used = out->n_gpu ? f[6] : 0.0;
  out->sum_resv = f[3]; out->max_resv = out->n_gpu ? f[7] : 0.0;
  out->max_total = out->n_gpu ? f[8] : 0.0;
  out->max_ratio = (f[9] > -INFINITY) ? f[9] : -1.0;
  out->ts_max = f[10]; out->ts_min = -f[11];
  out->max_cores = (u32)f[12];
  out->any_gpu_available = f[13] > 0.5 ? 1u : 0u;
  return TML_OK;
}

int tml_proc_reduce(tml_ctx* c, uint32_t max_rows, void* stream, tml_proc_agg* out) {
  if (!c || !out || max_rows == 0) return TML_ERR_ARG;
  int rc = tml_proc_reduce_launch(c, max_rows, stream);
  if (rc != TML_OK) return rc;
  CK(cudaStreamSynchronize((cudaStream_t)stream));
  return tml_proc_reduce_collect(c, out);
}

}  // extern "C"

#include "tml_combined.cuh"
