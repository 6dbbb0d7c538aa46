// tml_sys_sum.h -- the float arithmetic of the System reduce (K6s, k_sys_reduce), shared by the
// kernel and its host emulation (tml_sys_host_sum), so the CPU suite fuzzes the code the GPU runs.
//
// The reference averages with CPython 3.12's sum() (compensated: Neumaier's variant of
// Kahan-Babuska) divided by len():
//   per sample  aggregator/sqlite_writers/system.py:459-474 -- <= 16 GPU values: SysCpySum
//               restates CPython's loop term by term, so the result is the same double by
//               construction;
//   per window  reporting/sections/system/model.py:189-192 -- up to 10^5 terms: a TwoSum
//               double-double carried through every level of the reduction tree and rounded once.
//               Integer-valued columns (bytes, %, deg C) are summed exactly as u64 instead.
// Build with -fmad=false: a contracted a*b+c would change the error terms.
//
// The sample-level window columns travel between the two steps of every reduction as a
// tml_sys_part: K6s folds its CTA partials (sys_part_merge, in CTA order) and rounds once
// (sys_part_finish); K6m folds the nodes' parts in the reference's row order and rounds once the
// same way (sys_cluster_fold), so the cluster rollup is the window sum over all nodes' samples.
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define TML_SYS_HD __host__ __device__ __forceinline__
#else
#define TML_SYS_HD inline
#endif

#define SYS_THREADS 256  // k_sys_reduce block size: 8 warps

// CPython 3.12 builtin_sum_impl over floats with the default int start: the first item becomes the
// running float (0 + x == x), every later item goes through Neumaier's update, and the
// compensation is added once at the end when it is non-zero and finite.
struct SysCpySum {
  double f, c;
  int k;
  TML_SYS_HD void init() { f = 0.0; c = 0.0; k = 0; }
  TML_SYS_HD void add(double x) {
    if (k++ == 0) { f = x; return; }
    const double t = f + x;
    const double af = f < 0.0 ? -f : f, ax = x < 0.0 ? -x : x;
    if (af >= ax) c += (f - t) + x;
    else c += (x - t) + f;
    f = t;
  }
  TML_SYS_HD double value() const { return (c != 0.0 && c - c == 0.0) ? f + c : f; }  // c - c == 0: finite
};

TML_SYS_HD double sys_cpython_sum(const double* x, uint64_t n) {
  SysCpySum s;
  s.init();
  for (uint64_t i = 0; i < n; ++i) s.add(x[i]);
  return s.value();
}

// TwoSum accumulate of (xh, xl) into the unevaluated pair (hi, lo); the value is hi + lo.
TML_SYS_HD void sys_dd_add(double& hi, double& lo, double xh, double xl) {
  const double s = hi + xh;
  const double bp = s - hi;
  const double err = (hi - (s - bp)) + (xh - bp);
  hi = s;
  lo = (lo + xl) + err;
}

// The derived columns of one sample (system.py:459-474), over its first n >= 1 GPU entries in
// index order: d[0] util avg, d[1] util peak, d[2] mem avg, d[3] mem peak, d[4] temp avg,
// d[5] temp peak, d[6] power avg (W), d[7] power peak (W).  Peaks are max() of the same floats.
TML_SYS_HD void sys_derive(const tml_sys_gpu* g, int n, double d[8]) {
  SysCpySum su, sm, st, sp;
  su.init(); sm.init(); st.init(); sp.init();
  double um = 0.0, mm = 0.0, tm = 0.0, pm = 0.0;
  for (int i = 0; i < n; ++i) {
    const double u = (double)g[i].util, m = (double)g[i].mem_used, t = (double)g[i].temp_c;
    const double p = (double)g[i].power_mw / 1000.0;  // SystemProbe: nvmlDeviceGetPowerUsage(h) / 1000.0
    su.add(u); sm.add(m); st.add(t); sp.add(p);
    if (i == 0 || u > um) um = u;
    if (i == 0 || m > mm) mm = m;
    if (i == 0 || t > tm) tm = t;
    if (i == 0 || p > pm) pm = p;
  }
  const double len = (double)n;
  d[0] = su.value() / len; d[1] = um;
  d[2] = sm.value() / len; d[3] = mm;
  d[4] = st.value() / len; d[5] = tm;
  d[6] = sp.value() / len; d[7] = pm;
}

TML_SYS_HD uint64_t sys_max_u64(uint64_t a, uint64_t b) { return a > b ? a : b; }
TML_SYS_HD uint32_t sys_max_u32(uint32_t a, uint32_t b) { return a > b ? a : b; }

TML_SYS_HD void sys_part_init(tml_sys_part& a) {
  a.cpu_hi = a.cpu_lo = 0.0; a.cpu_max = -INFINITY; a.ts_min = INFINITY; a.ts_max = -INFINITY;
  for (int k = 0; k < 4; ++k) { a.d_hi[k] = 0.0; a.d_lo[k] = 0.0; a.d_max[k] = -INFINITY; }
  a.ram_sum = a.ram_max = a.ram_total_max = a.n = a.n_gpu = 0;
  a.avail = a.gpu_count = a.n_gpus = a._pad = 0;
}

// Fold b into a.  Order matters only for the double-double sums (each step is a TwoSum).
TML_SYS_HD void sys_part_merge(tml_sys_part& a, const tml_sys_part& b) {
  sys_dd_add(a.cpu_hi, a.cpu_lo, b.cpu_hi, b.cpu_lo);
  a.cpu_max = fmax(a.cpu_max, b.cpu_max); a.ts_min = fmin(a.ts_min, b.ts_min); a.ts_max = fmax(a.ts_max, b.ts_max);
  for (int k = 0; k < 4; ++k) { sys_dd_add(a.d_hi[k], a.d_lo[k], b.d_hi[k], b.d_lo[k]); a.d_max[k] = fmax(a.d_max[k], b.d_max[k]); }
  a.ram_sum += b.ram_sum; a.ram_max = sys_max_u64(a.ram_max, b.ram_max);
  a.ram_total_max = sys_max_u64(a.ram_total_max, b.ram_total_max);
  a.n += b.n; a.n_gpu += b.n_gpu;
  a.avail |= b.avail; a.gpu_count = sys_max_u32(a.gpu_count, b.gpu_count); a.n_gpus = sys_max_u32(a.n_gpus, b.n_gpus);
}

// Round a fold once into the sample-level fields of tml_sys_agg (loader.py:97-125); the per-GPU
// rows are left as they are.
TML_SYS_HD void sys_part_finish(const tml_sys_part& b, tml_sys_agg* out) {
  const double cnt = (double)b.n;
  out->n = b.n; out->n_gpu = b.n_gpu;
  out->first_ts = b.ts_min; out->last_ts = b.ts_max;
  out->cpu_avg = (b.cpu_hi + b.cpu_lo) / cnt; out->cpu_peak = b.cpu_max;
  out->ram_avg = (double)b.ram_sum / cnt; out->ram_peak = (double)b.ram_max;
  out->ram_total = (double)b.ram_total_max;
  const double cg = (double)b.n_gpu;
  const bool hg = b.n_gpu > 0;
  out->gpu_util_avg = hg ? (b.d_hi[0] + b.d_lo[0]) / cg : 0.0; out->gpu_util_peak = hg ? b.d_max[0] : 0.0;
  out->gpu_mem_avg = hg ? (b.d_hi[1] + b.d_lo[1]) / cg : 0.0; out->gpu_mem_peak = hg ? b.d_max[1] : 0.0;
  out->gpu_temp_avg = hg ? (b.d_hi[2] + b.d_lo[2]) / cg : 0.0; out->gpu_temp_peak = hg ? b.d_max[2] : 0.0;
  out->gpu_power_avg = hg ? (b.d_hi[3] + b.d_lo[3]) / cg : 0.0; out->gpu_power_peak = hg ? b.d_max[3] : 0.0;
  out->gpu_available = b.avail; out->gpu_count = b.gpu_count; out->n_gpus = b.n_gpus; out->_pad = 0;
}

// The node label as an integer (loader.py:78-81): node_rank, else global_rank.
TML_SYS_HD int64_t sys_node_key(const tml_sys_node_ident& id) {
  return id.node_rank >= 0 ? (int64_t)id.node_rank : (int64_t)id.global_rank;
}

// K6m's whole computation (one thread): pick the valid records, one per label (the lowest global
// rank), order them by (label, global rank) ascending -- the reference's cluster rows are ordered
// by COALESCE(node_rank, global_rank) -- fold their parts in that order and round once.
TML_SYS_HD void sys_cluster_fold(const tml_sys_node_record* rec, uint32_t n, tml_sys_cluster_out* out) {
  uint32_t used = 0, dup = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (!rec[i].valid) continue;
    const int64_t key = sys_node_key(rec[i].ident);
    bool keep = true;
    for (uint32_t j = 0; j < n && keep; ++j) {
      if (j == i || !rec[j].valid || sys_node_key(rec[j].ident) != key) continue;
      const int32_t gi = rec[i].ident.global_rank, gj = rec[j].ident.global_rank;
      if (gj < gi || (gj == gi && j < i)) keep = false;
    }
    if (!keep) { ++dup; continue; }
    uint32_t at = used++;  // insertion sort by (key, global rank)
    while (at > 0) {
      const tml_sys_node_ident& p = rec[out->order[at - 1]].ident;
      const int64_t pk = sys_node_key(p);
      if (pk < key || (pk == key && p.global_rank < rec[i].ident.global_rank)) break;
      out->order[at] = out->order[at - 1];
      --at;
    }
    out->order[at] = (int32_t)i;
  }
  for (uint32_t k = used; k < TML_MAX_RANKS; ++k) out->order[k] = -1;
  tml_sys_part b;
  sys_part_init(b);
  for (uint32_t k = 0; k < used; ++k) sys_part_merge(b, rec[out->order[k]].part);
  tml_sys_agg* a = &out->agg;
  char* z = (char*)a;
  for (size_t k = 0; k < sizeof(tml_sys_agg); ++k) z[k] = 0;
  if (used) sys_part_finish(b, a);
  out->n_nodes = used;
  out->n_dup = dup;
}
