// tml_exact_sum_host.cpp -- serial host emulation of K3e (tml_exact_sum.cuh) for ONE chain.
// TEST HOOK: lets the CPU suite fuzz the monoid arithmetic of tml_exact_sum.h -- plan, chunk /
// group composition, verified application, tile fallback -- against a plain sequential loop
// without a GPU.  The product never calls it; the GPU kernels share the header, not this file.
#include <cstdint>
#include <vector>

#include "../../include/traceml_b200.h"
#include "tml_exact_sum.h"

extern "C" int tml_xs_host_sum(const double* x, uint64_t n, int planned, double* out_sum, uint64_t* slow_rows) {
  if ((!x && n) || !out_sum) return TML_ERR_ARG;
  const uint64_t nchunks = (n + XS_CHUNK - 1) / XS_CHUNK, ngroups = (nchunks + XS_GROUP - 1) / XS_GROUP;
  std::vector<double> csum(nchunks, 0.0);
  std::vector<int> plan(nchunks, XS_PLAN_UNSAFE), gplan(ngroups, XS_PLAN_UNSAFE);
  std::vector<XsFn> fn(nchunks, xs_invalid()), gfn(ngroups, xs_invalid());
  if (planned) {
    for (uint64_t c = 0; c < nchunks; ++c) {  // X1: any summation order will do (approximate)
      double a = 0.0;
      const uint64_t lo = c * XS_CHUNK, hi = lo + XS_CHUNK < n ? lo + XS_CHUNK : n;
      for (uint64_t i = hi; i > lo; --i) a += x[i - 1];
      csum[c] = a;
    }
    double run = 0.0;  // X2
    for (uint64_t c = 0; c < nchunks; ++c) { plan[c] = xs_plan(run, run + csum[c]); run += csum[c]; }
    for (uint64_t c = 0; c < nchunks; ++c) {  // X3
      if (plan[c] == XS_PLAN_ZERO) { fn[c] = xs_identity(); continue; }
      if (plan[c] < 1) continue;
      XsFn f = xs_identity();  // the kernels' hot loop: FPU element maps, raw compose, sealed once per chunk
      bool ok = true;
      const double scale = xs_scale(plan[c]);
      const uint64_t lo = c * XS_CHUNK, hi = lo + XS_CHUNK < n ? lo + XS_CHUNK : n;
      for (uint64_t i = lo; i < hi; ++i) {
        XsFn g, gi;
        ok = xs_elem_fp(x[i], plan[c], scale, &g) && ok;
        const bool oki = xs_elem_raw(x[i], plan[c], &gi);  // the integer formulation must agree, always
        if (oki && (g.c0 != gi.c0 || g.c1 != gi.c1)) return TML_ERR_STATE;
        if (oki && scale != 0.0) {  // and so must the branch-free forms of the compose kernel
          bool bad = false;
          const XsFn gn = xs_elem_fp_nb(x[i], scale, &bad);
          const XsFn h1 = xs_compose_raw(f, g), h2 = xs_compose_nb(f, gn);
          if (bad || gn.c0 != gi.c0 || gn.c1 != gi.c1 || h1.c0 != h2.c0 || h1.c1 != h2.c1) return TML_ERR_STATE;
        }
        f = xs_compose_raw(f, g);
      }
      fn[c] = xs_seal(f, ok);
    }
    for (uint64_t g = 0; g < ngroups; ++g) {  // X3b
      int emax = XS_PLAN_ZERO;
      const uint64_t lo = g * XS_GROUP, hi = lo + XS_GROUP < nchunks ? lo + XS_GROUP : nchunks;
      for (uint64_t c = lo; c < hi; ++c) emax = plan[c] > emax ? plan[c] : emax;
      bool ok = emax >= 1;
      XsFn f = xs_identity();
      for (uint64_t c = lo; c < hi; ++c) {
        ok = ok && (plan[c] == emax || plan[c] == XS_PLAN_ZERO);
        f = xs_compose(f, fn[c]);
      }
      gfn[g] = ok ? f : xs_invalid();
      gplan[g] = emax == XS_PLAN_ZERO ? XS_PLAN_ZERO : (ok ? emax : XS_PLAN_UNSAFE);
    }
  }
  double s = 0.0;
  uint64_t slow = 0;
  for (uint64_t g = 0; g < ngroups; ++g) {  // X4
    if (gplan[g] == XS_PLAN_ZERO) continue;
    {
      int eb; unsigned long long S;
      xs_unpack(s, &eb, &S);
      if (gplan[g] >= 1 && xs_apply_s(eb, &S, gfn[g], gplan[g])) { s = xs_pack(eb, S); continue; }
    }
    const uint64_t clo = g * XS_GROUP, chi = clo + XS_GROUP < nchunks ? clo + XS_GROUP : nchunks;
    for (uint64_t c = clo; c < chi; ++c) {
      if (plan[c] == XS_PLAN_ZERO) continue;
      if (plan[c] >= 1 && xs_apply(&s, fn[c], plan[c])) continue;
      const uint64_t lo = c * XS_CHUNK, hi = lo + XS_CHUNK < n ? lo + XS_CHUNK : n;
      for (uint64_t t = lo; t < hi; t += 32) {
        const uint64_t te = t + 32 < hi ? t + 32 : hi;
        const int eb = xs_exp(s);
        bool done = false;
        if (eb >= 1 && eb < 0x7ff && s > 0.0) {
          XsFn f = xs_identity();
          for (uint64_t i = t; i < te; ++i) f = xs_compose(f, xs_elem(x[i], eb));
          done = xs_apply(&s, f, eb);
        }
        if (!done) {
          for (uint64_t i = t; i < te; ++i) s += x[i];
          slow += te - t;
        }
      }
    }
  }
  *out_sum = s;
  if (slow_rows) *slow_rows = slow;
  return TML_OK;
}

// ---------------------------------------------------------------------------------------------
// Host emulation of k_sys_reduce's float sums (tml_sys_sum.h): mode 0 the per-sample CPython
// restatement, mode 1 the window's double-double through the kernel's tree -- grid-stride
// threads of nblk CTAs, warp butterfly (lane l merges lane l ^ m, m = 16 .. 1), the eight warps
// in order, then the CTA partials in order -- rounded once.
#include "tml_sys_sum.h"

extern "C" int tml_sys_host_sum(const double* x, uint64_t n, uint32_t mode, uint32_t nblk, double* out_sum) {
  if ((!x && n) || !out_sum || mode > 2) return TML_ERR_ARG;
  if (mode == 0) { *out_sum = sys_cpython_sum(x, n); return TML_OK; }
  if (nblk == 0) return TML_ERR_ARG;
  double gh = 0.0, gl = 0.0;
  for (uint32_t b = 0; b < nblk; ++b) {
    double th[SYS_THREADS], tl[SYS_THREADS];
    for (int t = 0; t < SYS_THREADS; ++t) {
      th[t] = 0.0; tl[t] = 0.0;
      for (uint64_t i = (uint64_t)b * SYS_THREADS + t; i < n; i += (uint64_t)nblk * SYS_THREADS)
        sys_dd_add(th[t], tl[t], x[i], 0.0);
    }
    double bh = 0.0, bl = 0.0;
    for (int w = 0; w < SYS_THREADS / 32; ++w) {
      double h[32], l[32];
      for (int k = 0; k < 32; ++k) { h[k] = th[w * 32 + k]; l[k] = tl[w * 32 + k]; }
      for (int m = 16; m >= 1; m >>= 1) {
        double nh[32], nl[32];
        for (int k = 0; k < 32; ++k) { nh[k] = h[k]; nl[k] = l[k]; sys_dd_add(nh[k], nl[k], h[k ^ m], l[k ^ m]); }
        for (int k = 0; k < 32; ++k) { h[k] = nh[k]; l[k] = nl[k]; }
      }
      sys_dd_add(bh, bl, h[0], l[0]);
    }
    sys_dd_add(gh, gl, bh, bl);
  }
  if (mode == 2) { out_sum[0] = gh; out_sum[1] = gl; return TML_OK; }
  *out_sum = gh + gl;
  return TML_OK;
}

extern "C" int tml_sys_host_cluster(const tml_sys_node_record* records, uint32_t n_records, tml_sys_cluster_out* out) {
  if ((!records && n_records) || !out || n_records > TML_MAX_RANKS) return TML_ERR_ARG;
  sys_cluster_fold(records, n_records, out);
  return TML_OK;
}
