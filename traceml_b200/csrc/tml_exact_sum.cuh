// tml_exact_sum.cuh -- K3e: the seven per-rank window sums in the REFERENCE'S summation order,
// bit for bit, for any window size (math and rationale: tml_exact_sum.h).  Included by
// tml_engine.cu; replaces round 1's single-thread dependency chain (k_seq_sums, <= 2^17 rows).
//
// Work unit: a CHUNK of 256 consecutive rows (in summation order) = one warp of the compose kernel;
// 32 chunks = one GROUP.  Maps compose associatively, so every level is built in parallel and only
// the walk -- a few hundred map applications plus one 32-row tile per binade crossing -- is serial.
//
//   X1 k_xs_prefix    running prefix of the approximate chunk sums K3a left in the workspace
//      (k_xs_partial  computes those sums in a pass of its own: aligned sources, TML_XS_K3A_CSUM=0)
//   X2 k_xs_bscan     exclusive scan of the CTA totals (one small CTA)
//   X3 k_xs_compose   chunk -> exponent plan + 7 (c0, c1) maps; for a chunk whose running sum
//                     changes binade: the eight 32-row TILE maps under both candidate exponents
//   X3b k_xs_groups   32 chunks -> one map (warp-ordered composition)
//   X4 k_xs_walk      one CTA per chain: groups -> chunks -> tiles, 32 maps per warp step; only the
//                     tile that contains a binade crossing (and the start-up from 0) is redone with
//                     real adds
//
// Window sums read the rows once (X3: 64 B/row; the chunk sums come out of K3a's registers), aligned
// sums twice.  At R > 1 K3e runs beside the NVLink-bound K4 on a side stream; the R = 1 bulk path
// does not need reference-order sums at all (no second rank to break a tie against) and skips K3e.
#pragma once
#include "tml_exact_sum.h"

#define XS_WARPS 8                       // chunks per CTA trip
#define XS_ROWS_PER_LANE (XS_CHUNK / 32)  // 8
#define XS_TILES (XS_CHUNK / 32)          // 32-row tiles per chunk (= 4 lanes each)
#define XS_SLOT_CAP 4096                  // (chunk, chain) pairs that may carry tile maps
#define XS_PLAN_SLOT0 (-3)                // plan <= XS_PLAN_SLOT0: unsafe, tile maps in slot -(plan) - 3

struct XsSrc {
  const tml_window_row* rows;
  const u8* flags;      // window mode: only rows with (flags & need) == need count; others add +0.0
  u32 need;
  long long first, last;  // inclusive; summation order is last, last - 1, ..., first (newest row first)
  int aligned;            // 1: addend 4 is max(0, traced) (alignment.py:72), 0: the step wall (model.py:265)
  const tml_window_row* xrows;  // aligned mode: where the aligned rows live is decided on the device
  const u32* noncontig;
  const u32* sel_rows;
  long long dense_first;
  long long pad;          // leading virtual +0.0 positions: summation position p reads row last - (p - pad).
                          // Window mode pads so that chunk boundaries fall on row indices that are
                          // multiples of 256 -- then K3a's 32-row tiles never straddle a chunk and K3a
                          // itself can deliver the approximate chunk sums (no separate pass over the rows)
};

struct XsTileMaps {  // one unsafe (chunk, chain): tile maps under exponent ea (h = 0) and ea + 1 (h = 1)
  XsFn f[2][XS_TILES];
  double x[XS_CHUNK];  // and the chain's addends, in summation order: the crossing tile is added from here
};
struct XsTileHead { XsFn f[2][XS_TILES]; };  // the part of a slot the walk stages in shared memory

struct XsWork {  // device workspace of one launch
  double* csum;   // [nchunks][8] approximate chunk sums
  double* cpre;   // [nchunks][8] their exclusive prefix inside the owning CTA's run
  double* btot;   // [nblocks][8]
  double* bpre;   // [nblocks][8]
  int* plan;      // [nchunks][8]
  int* ea;        // [nchunks][8] candidate exponent of an unsafe chunk (tile maps: ea, ea + 1)
  XsFn* fn;       // [nchunks][7]
  XsFn* gfn;      // [ngroups][7]
  int* gplan;     // [ngroups][8]
  XsTileMaps* tiles;  // [XS_SLOT_CAP]
  unsigned int* nslots;
};

__device__ __forceinline__ const tml_window_row* xs_rows(const XsSrc& s) {
  if (!s.aligned) return s.rows;
  if (s.dense_first >= 0) return s.rows + s.dense_first;
  return (*s.noncontig) ? s.xrows : (s.rows + s.sel_rows[0]);
}

// One row of summation position p (p = 0 is the newest row), in two steps so that a caller can
// put the loads of several rows in flight before it touches any of them: xs_row_load issues the
// flag and row loads (no branch depends on what they return), xs_row_addends turns them into the
// seven addends -- zeros past the end or for a row the section does not use.
struct XsRowRaw { uint4 a, b, c; unsigned fl; bool in; };

__device__ __forceinline__ XsRowRaw xs_row_load(const tml_window_row* __restrict__ rows, const XsSrc& s, long long p,
                                                long long n) {
  XsRowRaw r;
  r.a = r.b = r.c = make_uint4(0u, 0u, 0u, 0u);
  r.fl = 0u;
  p -= s.pad;
  r.in = (p >= 0 && p < n - s.pad);
  if (r.in) {
    const long long i = s.last - p;
    if (s.flags) r.fl = s.flags[i];
    const uint4* src = reinterpret_cast<const uint4*>(rows + i);
    r.a = __ldg(src); r.b = __ldg(src + 1); r.c = __ldg(src + 2);
  }
  return r;
}

__device__ __forceinline__ void xs_row_addends(const XsRowRaw& r, const XsSrc& s, double (&o)[7]) {
  const bool keep = r.in && (!s.flags || ((r.fl & s.need) == s.need));
  const double dl = __longlong_as_double((long long)((u64)r.a.x | ((u64)r.a.y << 32)));
  const double fwd = __longlong_as_double((long long)((u64)r.b.x | ((u64)r.b.y << 32)));
  const double bwd = __longlong_as_double((long long)((u64)r.b.z | ((u64)r.b.w << 32)));
  const double opt = __longlong_as_double((long long)((u64)r.c.x | ((u64)r.c.y << 32)));
  const double wall = __longlong_as_double((long long)((u64)r.c.z | ((u64)r.c.w << 32)));
  const double compute = (fwd + bwd) + opt;
  const double traced = fmax(wall, compute);
  o[0] = dl; o[1] = fwd; o[2] = bwd; o[3] = opt;
  o[4] = s.aligned ? fmax(0.0, traced) : wall;
  o[5] = traced;
  o[6] = dl + traced;
  if (!keep) {
#pragma unroll
    for (int k = 0; k < 7; ++k) o[k] = 0.0;
  }
}

// the seven addends of summation position p; zeros past the end
__device__ __forceinline__ void xs_addends(const tml_window_row* __restrict__ rows, const XsSrc& s, long long p,
                                           long long n, double (&o)[7]) {
  const XsRowRaw r = xs_row_load(rows, s, p, n);
  xs_row_addends(r, s, o);
}

__device__ __forceinline__ double xs_pick(const double (&o)[7], int k) {
  double x = o[0];
#pragma unroll
  for (int m = 1; m < 7; ++m) x = (k == m) ? o[m] : x;
  return x;
}

__device__ __forceinline__ u64 shfl_down_u64(u64 v, int d) { return __shfl_down_sync(0xffffffffu, v, d); }

// ordered composition over the warp: lane 0 receives f[0] o f[1] o ... o f[31] (f[0] applied first);
// after the levels d = 1, 2 lanes 0, 4, 8, ... hold the maps of their 4-lane group (one 32-row tile)
__device__ __forceinline__ XsFn xs_warp_compose(XsFn f, int lane, XsFn* tile_out = nullptr) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    XsFn g;
    g.c0 = shfl_down_u64(f.c0, d);
    g.c1 = shfl_down_u64(f.c1, d);
    if ((lane & (2 * d - 1)) == 0) f = xs_compose(f, g);
    if (d == 2 && tile_out) *tile_out = f;
  }
  return f;
}

// same tree on unsealed maps (callers seal lane 0's result)
__device__ __forceinline__ XsFn xs_warp_compose_raw(XsFn f, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    XsFn g;
    g.c0 = shfl_down_u64(f.c0, d);
    g.c1 = shfl_down_u64(f.c1, d);
    if ((lane & (2 * d - 1)) == 0) f = xs_compose_raw(f, g);
  }
  return f;
}

__device__ __forceinline__ void xs_block_range(long long nchunks, long long* lo, long long* hi) {
  long long per = (nchunks + gridDim.x - 1) / gridDim.x;
  per = (per + XS_WARPS - 1) / XS_WARPS * XS_WARPS;
  *lo = (long long)blockIdx.x * per;
  *hi = (*lo + per < nchunks) ? *lo + per : nchunks;
}

// ---- X1
__global__ void __launch_bounds__(XS_WARPS * 32) k_xs_partial(const XsSrc s, long long n, long long nchunks, XsWork w) {
  __shared__ double s_part[XS_WARPS][7];
  const tml_window_row* rows = xs_rows(s);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  long long c_lo, c_hi;
  xs_block_range(nchunks, &c_lo, &c_hi);
  double run = 0.0;  // threads 0..6: running prefix of chain `threadIdx.x` inside this CTA's run
  for (long long base = c_lo; base < c_hi; base += XS_WARPS) {
    const long long ch = base + warp;
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    if (ch < c_hi) {
#pragma unroll
      for (int j = 0; j < XS_ROWS_PER_LANE; ++j) {
        double o[7];
        xs_addends(rows, s, ch * XS_CHUNK + lane * XS_ROWS_PER_LANE + j, n, o);
#pragma unroll
        for (int k = 0; k < 7; ++k) acc[k] += o[k];
      }
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      double x = acc[k];
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) x += shfl_xor_f64(x, m);
      if (lane == 0) s_part[warp][k] = x;
    }
    __syncthreads();
    if (threadIdx.x < 7) {
#pragma unroll
      for (int q = 0; q < XS_WARPS; ++q) {
        if (base + q < c_hi) {
          const double v = s_part[q][threadIdx.x];
          w.cpre[(base + q) * 8 + threadIdx.x] = run;
          w.csum[(base + q) * 8 + threadIdx.x] = v;
          run += v;
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x < 7) w.btot[(long long)blockIdx.x * 8 + threadIdx.x] = run;
}

// ---- X1': the chunk sums are already there (K3a accumulated them while it had the rows in
// registers): only the running prefix inside each CTA's run and the CTA totals remain
__global__ void __launch_bounds__(32) k_xs_prefix(long long nchunks, XsWork w) {
  long long c_lo, c_hi;
  xs_block_range(nchunks, &c_lo, &c_hi);
  if (threadIdx.x < 7) {
    double run = 0.0;
    for (long long ch = c_lo; ch < c_hi; ++ch) {
      const double v = w.csum[ch * 8 + threadIdx.x];
      w.cpre[ch * 8 + threadIdx.x] = run;
      run += v;
    }
    w.btot[(long long)blockIdx.x * 8 + threadIdx.x] = run;
  }
}

// ---- X2: exclusive scan of the CTA totals (one CTA, tiles of 1024 with a running carry)
__global__ void __launch_bounds__(1024) k_xs_bscan(XsWork w, int nblocks) {
  __shared__ double s_warp[32][7];
  __shared__ double s_carry[7];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  if (t < 7) s_carry[t] = 0.0;
  __syncthreads();
  for (int base = 0; base < nblocks; base += 1024) {
    const int i = base + t;
    double v[7], excl[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      v[k] = (i < nblocks) ? w.btot[(long long)i * 8 + k] : 0.0;
      double incl = v[k];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        double y = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += y;
      }
      if (lane == 31) s_warp[warp][k] = incl;
      excl[k] = incl - v[k];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        double x = s_warp[lane][k], incl = x;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          double y = __shfl_up_sync(0xffffffffu, incl, off);
          if (lane >= off) incl += y;
        }
        s_warp[lane][k] = incl - x;
      }
    }
    __syncthreads();
    double tot[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const double pre = s_carry[k] + s_warp[warp][k] + excl[k];
      if (i < nblocks) w.bpre[(long long)i * 8 + k] = pre;
      tot[k] = pre + v[k];
    }
    __syncthreads();
    if (t == 1023) {
#pragma unroll
      for (int k = 0; k < 7; ++k) s_carry[k] = tot[k];
    }
    __syncthreads();
  }
  if (t == 0) *w.nslots = 0u;
}

// ---- X3.  One warp per chunk.  Phase A: lane = row (two passes of four rows per lane, the flag and
// row loads of a pass all in flight before the first is used); the seven addends of a row are
// derived ONCE and parked in shared memory, chain by chain.  Phase B: lane = (g, k), row quarter
// g = lane >> 3 (64 consecutive rows), chain k = lane & 7 (k == 7 idles): a lane walks its 64 rows
// serially for ITS chain -- one LDS, one branch-free FPU element map, one branch-free compose per
// row -- and the four quarters of a chain are joined by two shuffle levels.  Deriving the addends
// once in shared memory, instead of every lane deriving all seven from global memory, cuts the
// warp instructions several-fold.
#define XS_CW 2                    // warps (chunks in flight) per compose CTA
#define XS_SG 65                   // doubles per row quarter (64 + 1: quarters in different banks)
#define XS_SK (4 * XS_SG + 8)      // doubles per chain

__global__ void __launch_bounds__(XS_CW * 32) k_xs_compose(const XsSrc s, long long n, long long nchunks, XsWork w,
                                                          int chunks_per_block) {
  __shared__ double s_x[XS_CW][7 * XS_SK];
  const tml_window_row* rows = xs_rows(s);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 3, k = lane & 7;
  const bool live = k < 7;
  double* sm = s_x[warp];
  // this CTA serves the chunks [blockIdx.x * XS_CW, +XS_CW); the prefix tables are indexed by the
  // CTA that PRODUCED them in X1 (runs of `chunks_per_block` chunks)
  const long long ch = (long long)blockIdx.x * XS_CW + warp;
  if (ch >= nchunks) return;
  const long long owner = ch / chunks_per_block;
  double lo = 0.0;
  int e = XS_PLAN_ZERO;
  if (live) {
    lo = w.bpre[owner * 8 + k] + w.cpre[ch * 8 + k];
    e = xs_plan(lo, lo + w.csum[ch * 8 + k]);
  }
  // ---- phase A: four rows per lane in flight (flags + 3 x 16 B each) before the first is used
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    XsRowRaw raw[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      raw[q] = xs_row_load(rows, s, ch * XS_CHUNK + (half * 4 + q) * 32 + lane, n);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int r = (half * 4 + q) * 32 + lane;
      double o[7];
      xs_row_addends(raw[q], s, o);
      double* dst = sm + (r >> 6) * XS_SG + (r & 63);
#pragma unroll
      for (int m = 0; m < 7; ++m) dst[m * XS_SK] = o[m];
    }
  }
  __syncwarp();
  // ---- phase B
  const double* mine = sm + (live ? k : 0) * XS_SK + g * XS_SG;
  double scale = e >= 1 ? xs_scale(e) : 0.0;
  if (e >= 1 && scale == 0.0) e = XS_PLAN_UNSAFE;  // exponent without a normal scale (sums < 2^-971): walk adds rows
  XsFn f = xs_identity();
  bool bad = false;
  if (e >= 1) {
#pragma unroll 8
    for (int j = 0; j < 64; ++j) f = xs_compose_nb(f, xs_elem_fp_nb(mine[j], scale, &bad));
  }
  // join the four quarters of each chain: lanes k, k + 8, k + 16, k + 24 (in row order)
#pragma unroll
  for (int d = 8; d <= 16; d <<= 1) {
    XsFn m;
    m.c0 = shfl_down_u64(f.c0, d);
    m.c1 = shfl_down_u64(f.c1, d);
    const bool mbad = __shfl_down_sync(0xffffffffu, bad ? 1 : 0, d) != 0;
    if ((g & ((2 * d / 8) - 1)) == 0) { f = xs_compose_nb(f, m); bad = bad || mbad; }
  }
  if (live && g == 0) {
    XsFn r = xs_seal(f, !bad);  // 256 maps < 2^53 each: the raw sums stay < 2^61
    if (e == XS_PLAN_ZERO) r = xs_identity();
    else if (e < 1) r = xs_invalid();
    w.fn[ch * 7 + k] = r;
  }
  // a chunk whose running sum changes binade: the eight TILE maps under both candidate exponents +
  // the chain's addends, so the walk redoes only the one tile that holds the crossing (rare: about
  // one chunk per binade and chain)
  const bool unsafe = live && e == XS_PLAN_UNSAFE && lo > 0.0;
  int plan_out = e;
  if (__any_sync(0xffffffffu, unsafe)) {
    const int ea = unsafe ? xs_exp(lo * (1.0 - 1.0e-6)) : 0;
    const double sa = xs_scale(ea), sb = xs_scale(ea + 1);
    unsigned int slot = 0xffffffffu;
    if (unsafe && g == 0 && ea >= 1 && ea < 0x7fd && sa != 0.0 && sb != 0.0) slot = atomicAdd(w.nslots, 1u);
    slot = __shfl_sync(0xffffffffu, slot, k);  // from the chain's g == 0 lane
    if (unsafe && slot < XS_SLOT_CAP) {
#pragma unroll 1
      for (int half = 0; half < 2; ++half) {
        XsFn fa = xs_identity(), fb = xs_identity();
        bool bada = false, badb = false;
#pragma unroll 4
        for (int j = 0; j < 32; ++j) {
          const double x = mine[half * 32 + j];
          fa = xs_compose_nb(fa, xs_elem_fp_nb(x, sa, &bada));
          fb = xs_compose_nb(fb, xs_elem_fp_nb(x, sb, &badb));
          w.tiles[slot].x[g * 64 + half * 32 + j] = x;
        }
        w.tiles[slot].f[0][g * 2 + half] = xs_seal(fa, !bada);
        w.tiles[slot].f[1][g * 2 + half] = xs_seal(fb, !badb);
      }
      if (g == 0) { plan_out = XS_PLAN_SLOT0 - (int)slot; w.ea[ch * 8 + k] = ea; }
    }
  }
  if (live && g == 0) w.plan[ch * 8 + k] = plan_out;
}

// ---- X3b: one warp per (group, chain)
__global__ void __launch_bounds__(256) k_xs_groups(XsWork w, long long nchunks, long long ngroups) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (wid >= ngroups * 7) return;
  const long long g = wid / 7;
  const int k = (int)(wid % 7);
  const long long ch = g * XS_GROUP + lane;
  int e = XS_PLAN_ZERO;
  XsFn f = xs_identity();
  if (ch < nchunks) { e = w.plan[ch * 8 + k]; f = w.fn[ch * 7 + k]; }
  if (e <= XS_PLAN_SLOT0) e = XS_PLAN_UNSAFE;
  // one exponent for every non-zero chunk of the group, else the group is walked chunk by chunk
  int emax = e;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) { int y = __shfl_xor_sync(0xffffffffu, emax, m); emax = y > emax ? y : emax; }
  const bool ok = (e == emax) || (e == XS_PLAN_ZERO);
  const bool all_ok = __all_sync(0xffffffffu, ok) && emax >= 1;
  f = xs_warp_compose(f, lane);
  if (lane == 0) {
    w.gfn[g * 7 + k] = all_ok ? f : xs_invalid();
    w.gplan[g * 8 + k] = (emax == XS_PLAN_ZERO) ? XS_PLAN_ZERO : (all_ok ? emax : XS_PLAN_UNSAFE);
  }
}

// ---- X4: CTA k walks chain k.  The walk itself is one warp applying integer maps (every lane
// carries the same running sum: the updates are deterministic functions of broadcast values);
// the other warps only help to stage what it will need into shared memory -- all group maps of a
// batch, the chunk maps of the groups that cannot be applied whole, the tile maps of the chunks
// that cross a binade -- so that the dependent chain never waits on global memory except for the
// ~one 32-row tile per binade that is added row by row.
#define XS_GB 1024   // groups staged per batch
#define XS_IG 24     // groups of a batch whose chunk maps are staged (more: fetched on demand)
#define XS_TS 32     // crossing chunks of a batch whose tile maps are staged (more: on demand)

// Running sum of the walk as integers: s = S * 2^(eb - 1075); eb == 0 while s is still zero.
struct XsState { int eb; u64 S; };

__device__ __forceinline__ void xs_seq32(XsState* st, double x, u64* slow_rows) {
  double acc = st->eb ? xs_pack(st->eb, st->S) : 0.0;
#pragma unroll 8
  for (int r = 0; r < 32; ++r) acc += __shfl_sync(0xffffffffu, x, r);  // rows past n are +0.0
  xs_unpack(acc, &st->eb, &st->S);
  if (acc == 0.0) st->eb = 0;
  *slow_rows += 32;
}

// inclusive ordered scan over the warp: lane i receives m[0] o m[1] o ... o m[i] (m[0] applied
// first).  Raw maps: 32 sealed maps (< 2^53 each) stay below 2^58.
__device__ __forceinline__ XsFn xs_warp_scan_raw(XsFn m, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    XsFn p;
    p.c0 = __shfl_up_sync(0xffffffffu, m.c0, d);
    p.c1 = __shfl_up_sync(0xffffffffu, m.c1, d);
    if (lane >= d) m = xs_compose_raw(p, m);
  }
  return m;
}

// Apply entries [j, end) for as long as they apply; returns the first index that did not.  The
// whole warp works on 32 entries at a time: lane i composes entries j .. j+i (the maps are
// associative), applies that prefix to the running sum and the warp keeps the longest prefix that
// stays inside the binade -- the increments are non-negative, so "entry i overflows" is monotone in
// i and the result equals applying the entries one after the other.  `e` == nullptr: every entry
// was composed under exponent `e_all`.
__device__ __forceinline__ int xs_apply_run(XsState* st, const XsFn* __restrict__ f, const int* __restrict__ e,
                                            int e_all, int j, int end, int lane) {
  const int eb = st->eb;
  u64 S = st->S;
  while (j < end) {
    const int idx = j + lane;
    int E = XS_PLAN_ZERO;
    XsFn m = xs_identity();
    if (idx < end) { E = e ? e[idx] : e_all; m = f[idx]; }
    const bool zero = (E == XS_PLAN_ZERO);
    const bool ok = zero || (E == eb && E >= 1 && E < 0x7ff && m.c0 != ~0ull);
    const unsigned bad = __ballot_sync(0xffffffffu, !ok);
    const int nvalid = bad ? (__ffs(bad) - 1) : 32;
    if (zero || lane >= nvalid) m = xs_identity();
    const XsFn pre = xs_warp_scan_raw(m, lane);
    const u64 Si = S + ((S & 1ull) ? pre.c1 : pre.c0);
    const unsigned ov = __ballot_sync(0xffffffffu, (Si >> 53) != 0ull);
    int napply = ov ? (__ffs(ov) - 1) : 32;
    napply = napply < nvalid ? napply : nvalid;
    if (napply > 0) S = __shfl_sync(0xffffffffu, Si, napply - 1);
    j += napply;
    if (napply < 32) break;
  }
  st->S = S;
  return j < end ? j : end;
}

// one crossing chunk: tile maps `tm` (exponents ea, ea + 1) staged in shared memory, the chain's
// addends in the slot (global): only the tile that crosses is fetched and added row by row
__device__ __forceinline__ void xs_walk_tiles(const double* __restrict__ xraw, long long p0, long long n, int lane,
                                              const XsTileHead* tm, int ea, XsState* st, u64* slow_rows) {
  const long long left = (n - p0 + 31) / 32;
  const int nt = left < XS_TILES ? (int)left : XS_TILES;
  int t = 0;
#pragma unroll 1
  while (t < nt) {
    const int h = st->eb - ea;
    if (h == 0 || h == 1) {
      t = xs_apply_run(st, tm->f[h], nullptr, st->eb, t, nt, lane);
      if (t >= nt) break;
    }
    xs_seq32(st, xraw[t * 32 + lane], slow_rows);
    ++t;
  }
}

// a chunk without maps (start-up from 0, or the slot table was full)
__device__ __forceinline__ void xs_walk_rows(const tml_window_row* rows, const XsSrc& s, long long p0, long long n,
                                             int k, int lane, XsState* st, u64* slow_rows) {
  double x[XS_TILES];
#pragma unroll
  for (int t = 0; t < XS_TILES; ++t) {
    double o[7];
    xs_addends(rows, s, p0 + t * 32 + lane, n, o);
    x[t] = xs_pick(o, k);
  }
#pragma unroll
  for (int t = 0; t < XS_TILES; ++t) {
    if (p0 + t * 32 < n) {
      bool done = false;
      if (st->eb >= 1 && st->eb < 0x7ff && p0 > 0) {  // compose this tile under the true exponent
        XsFn f = xs_warp_compose(xs_elem(x[t], st->eb), lane);
        f.c0 = __shfl_sync(0xffffffffu, f.c0, 0); f.c1 = __shfl_sync(0xffffffffu, f.c1, 0);
        done = xs_apply_s(st->eb, &st->S, f, st->eb);
      }
      if (!done) xs_seq32(st, x[t], slow_rows);
    }
  }
}

// <= 64 registers: a walk CTA (16 K registers) must fit on an SM beside the resident K4 CTAs -- at
// 128 it does not, and on 8 ranks the walk then starts only when K4 has finished
__global__ void __launch_bounds__(256, 4) k_xs_walk(const XsSrc s, long long n, long long nchunks, long long ngroups,
                                                 XsWork w, int planned, double* __restrict__ out,
                                                 unsigned long long* __restrict__ stats /* [7]: rows added one by one */) {
  __shared__ XsFn s_g[XS_GB];
  __shared__ int s_ge[XS_GB];
  __shared__ int s_inv[XS_IG];
  __shared__ int s_ninv;
  __shared__ XsFn s_c[XS_IG + 1][XS_GROUP];      // row XS_IG: on-demand spare
  __shared__ int s_ce[XS_IG + 1][XS_GROUP];
  __shared__ short s_ts[XS_IG + 1][XS_GROUP];    // staged tile-map index of a crossing chunk, or -1
  __shared__ XsTileHead s_t[XS_TS + 1];          // entry XS_TS: on-demand spare
  __shared__ int s_tea[XS_TS + 1];
  __shared__ int s_tslot[XS_TS];                 // global slot of staged entry
  __shared__ int s_nts;
  const tml_window_row* rows = xs_rows(s);
  const int k = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  XsState st;
  st.eb = 0; st.S = 0ull;
  u64 slow_rows = 0;
  for (long long gb = 0; gb < ngroups; gb += XS_GB) {
    const int cnt = (int)((ngroups - gb) < XS_GB ? (ngroups - gb) : XS_GB);
    __syncthreads();
    // ---- stage 1: every group map of the batch
    for (int i = tid; i < cnt; i += blockDim.x) {
      XsFn gf = xs_invalid();
      int ge = XS_PLAN_UNSAFE;
      if (planned) { gf = w.gfn[(gb + i) * 7 + k]; ge = w.gplan[(gb + i) * 8 + k]; }
      s_g[i] = gf; s_ge[i] = ge;
    }
    __syncthreads();
    // ---- stage 2: which groups must be walked chunk by chunk (in order)
    if (warp == 0) {
      int ninv = 0;
      for (int base = 0; base < cnt; base += 32) {
        const bool bad = (base + lane < cnt) && s_ge[base + lane] == XS_PLAN_UNSAFE;
        const unsigned m = __ballot_sync(0xffffffffu, bad);
        const int pos = ninv + __popc(m & ((1u << lane) - 1u));
        if (bad && pos < XS_IG) s_inv[pos] = base + lane;
        ninv += __popc(m);
      }
      if (lane == 0) s_ninv = ninv < XS_IG ? ninv : XS_IG;
    }
    __syncthreads();
    const int ninv = s_ninv;
    for (int i = tid; i < ninv * XS_GROUP; i += blockDim.x) {
      const int gi = i / XS_GROUP, q = i % XS_GROUP;
      const long long ch = (gb + s_inv[gi]) * XS_GROUP + q;
      XsFn cf = xs_invalid();
      int ce = XS_PLAN_ZERO;  // past the end: nothing to add
      if (ch < nchunks) { ce = XS_PLAN_UNSAFE; if (planned) { cf = w.fn[ch * 7 + k]; ce = w.plan[ch * 8 + k]; } }
      s_c[gi][q] = cf; s_ce[gi][q] = ce; s_ts[gi][q] = -1;
    }
    __syncthreads();
    // ---- stage 3: tile maps of the crossing chunks among them
    if (warp == 0) {
      int nts = 0;
      for (int gi = 0; gi < ninv; ++gi) {
        const int ce = s_ce[gi][lane];
        const bool has = ce <= XS_PLAN_SLOT0;
        const unsigned m = __ballot_sync(0xffffffffu, has);
        const int pos = nts + __popc(m & ((1u << lane) - 1u));
        if (has && pos < XS_TS) { s_ts[gi][lane] = (short)pos; s_tslot[pos] = XS_PLAN_SLOT0 - ce; }
        nts += __popc(m);
      }
      if (lane == 0) s_nts = nts < XS_TS ? nts : XS_TS;
    }
    __syncthreads();
    const int nts = s_nts;
    for (int i = tid; i < nts * 2 * XS_TILES; i += blockDim.x) {
      const int ti = i / (2 * XS_TILES), e = i % (2 * XS_TILES);
      (&s_t[ti].f[0][0])[e] = (&w.tiles[s_tslot[ti]].f[0][0])[e];
    }
    for (int gi = tid / XS_GROUP; gi < ninv; gi += blockDim.x / XS_GROUP) {
      const int q = tid % XS_GROUP;
      const int ti = s_ts[gi][q];
      if (ti >= 0) s_tea[ti] = w.ea[((gb + s_inv[gi]) * XS_GROUP + q) * 8 + k];
    }
    __syncthreads();
    // ---- stage 4: the walk (warp 0)
    if (warp == 0) {
      int next_inv = 0;
      for (int j = 0; j < cnt; ++j) {
        j = xs_apply_run(&st, s_g, s_ge, 0, j, cnt, lane);
        if (j >= cnt) break;
        const long long c0 = (gb + j) * XS_GROUP;
        int gi = XS_IG;  // spare row
        if (next_inv < ninv && s_inv[next_inv] == j) {
          gi = next_inv++;
        } else {  // not staged (list overflow, or a planned map that did not apply): fetch now
          __syncwarp();
          const long long ch = c0 + lane;
          XsFn cf = xs_invalid();
          int ce = XS_PLAN_ZERO;
          if (ch < nchunks) { ce = XS_PLAN_UNSAFE; if (planned) { cf = w.fn[ch * 7 + k]; ce = w.plan[ch * 8 + k]; } }
          s_c[gi][lane] = cf; s_ce[gi][lane] = ce; s_ts[gi][lane] = -1;
          __syncwarp();
        }
        for (int q = 0; q < XS_GROUP; ++q) {
          q = xs_apply_run(&st, s_c[gi], s_ce[gi], 0, q, XS_GROUP, lane);
          if (q >= XS_GROUP) break;
          const int CE = s_ce[gi][q];
          const long long p0 = (c0 + q) * XS_CHUNK;
          if (p0 >= n) break;
          if (CE <= XS_PLAN_SLOT0) {
            int ti = s_ts[gi][q];
            if (ti < 0) {  // tile maps not staged: fetch now
              ti = XS_TS;
              __syncwarp();
              if (lane < 2 * XS_TILES) (&s_t[ti].f[0][0])[lane] = (&w.tiles[XS_PLAN_SLOT0 - CE].f[0][0])[lane];
              if (lane == 0) s_tea[ti] = w.ea[(c0 + q) * 8 + k];
              __syncwarp();
            }
            xs_walk_tiles(w.tiles[XS_PLAN_SLOT0 - CE].x, p0, n, lane, &s_t[ti], s_tea[ti], &st, &slow_rows);
          } else {
            xs_walk_rows(rows, s, p0, n, k, lane, &st, &slow_rows);
          }
        }
      }
    }
  }
  if (warp == 0 && lane == 0) { out[k] = st.eb ? xs_pack(st.eb, st.S) : 0.0; if (stats) stats[k] = slow_rows; }
}
