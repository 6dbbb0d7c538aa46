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
#pragma once

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
