// tml_sections_json: Step-Time / Step-Memory / Process sections of one reduce, as JSON.
//
// The native counterpart of traceml_b200/sections.py (build_step_time / build_step_memory /
// build_process + the O(R) public rollups): it consumes tml_reduce_run's output, runs the
// three rule engines (tml_diag_*) and emits exactly the objects sections.py builds, so the
// host does one JSON parse per final_summary() instead of interpreter work per section.
// Reference arithmetic followed (file:line under src/traceml/):
//   RankStepSummary from sums        reporting/sections/step_time/model.py:108-120,270-281
//   closest_rank_to_median           reporting/sections/step_time/model.py:77-105
//   wait average                     reporting/sections/step_time/model.py:284-307
//   global average / median / worst  reporting/sections/step_time/model.py:310-403
//   overview                         reporting/sections/step_time/model.py:445-498
//   step-memory rows / rollup        reporting/sections/step_memory/model.py:224-246,322-412
// sections.py stays as the specification; tests hold the two identical.

#include <algorithm>
#include <charconv>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/traceml_b200.h"
#include "tml_internal.h"

namespace {

typedef tml_json::Str S;  // arena-backed: see tml_internal.h

S jnum(double v) {
  if (!std::isfinite(v)) return "null";
  char buf[40];
  char* end = std::to_chars(buf, buf + 36, v).ptr;
  bool is_float = false;
  for (const char* p = buf; p < end; ++p) if (*p == '.' || *p == 'e' || *p == 'E' || *p == 'n') { is_float = true; break; }
  if (!is_float) { *end++ = '.'; *end++ = '0'; }
  return S(buf, end);
}
S jint(long long v) {
  char buf[24];
  return S(buf, std::to_chars(buf, buf + sizeof(buf), v).ptr);
}
S jq(const S& s) { return "\"" + s + "\""; }  // keys / labels here never need escaping
const S JNULL = "null";

struct Obj {
  S s;
  bool first = true;
  explicit Obj(size_t hint = 240) { s.reserve(hint); s += '{'; }
  Obj& kv(const char* k, size_t kn, const S& v) {
    if (!first) s += ',';
    first = false;
    s += '"'; s.append(k, kn); s += "\":"; s += v;
    return *this;
  }
  Obj& kv(const char* k, const S& v) { return kv(k, strlen(k), v); }
  Obj& kv(const S& k, const S& v) { return kv(k.data(), k.size(), v); }
  S done() { s += '}'; return std::move(s); }  // the object is spent afterwards
};

struct RankSummary {  // RankStepSummary
  int rank;
  long long n;
  double dl, fwd, bwd, opt, step_cpu, traced, compute, total;
};

RankSummary summary_from_sums(int rank, unsigned long long n, const double* s) {
  RankSummary r;
  const double d = (double)n;
  r.rank = rank; r.n = (long long)n;
  r.dl = s[0] / d; r.fwd = s[1] / d; r.bwd = s[2] / d; r.opt = s[3] / d;
  r.step_cpu = s[4] / d; r.traced = s[5] / d;
  r.compute = ((s[1] + s[2]) + s[3]) / d;
  r.total = s[6] / d;
  return r;
}
S summary_json(const RankSummary& r) {
  return Obj().kv("steps_analyzed", jint(r.n)).kv("avg_dataloader_ms", jnum(r.dl))
      .kv("avg_forward_ms", jnum(r.fwd)).kv("avg_backward_ms", jnum(r.bwd))
      .kv("avg_optimizer_ms", jnum(r.opt)).kv("avg_step_cpu_ms", jnum(r.step_cpu))
      .kv("avg_traced_step_ms", jnum(r.traced)).kv("avg_gpu_compute_ms", jnum(r.compute))
      .kv("avg_total_step_ms", jnum(r.total)).done();
}

double median_of(std::vector<double> v) {  // statistics.median
  std::sort(v.begin(), v.end());
  const size_t n = v.size(), m = n / 2;
  return (n & 1) ? v[m] : (v[m - 1] + v[m]) / 2.0;
}
// index (into ranks/vals, ascending rank order) of the rank closest to the median:
// tie-break |delta|, value, rank
int closest_to_median(const std::vector<int>& ranks, const std::vector<double>& vals) {
  const double med = median_of(vals);
  int best = 0;
  for (int i = 1; i < (int)vals.size(); ++i) {
    const double da = std::fabs(vals[i] - med), db = std::fabs(vals[best] - med);
    if (da < db || (da == db && (vals[i] < vals[best] || (vals[i] == vals[best] && ranks[i] < ranks[best]))))
      best = i;
  }
  return best;
}
// Python >= 3.12 builtin sum() over floats: Neumaier-compensated (Python/bltinmodule.c,
// _csum); the reference's rollups call it (model.py:345-352), so the last ulp follows it.
double py_sum(const std::vector<double>& v) {
  double total = 0.0, c = 0.0;
  for (double x : v) {
    const double t = total + x;
    if (std::fabs(total) >= std::fabs(x)) c += (total - t) + x; else c += (x - t) + total;
    total = t;
  }
  if (c != 0.0 && std::isfinite(c)) total += c;
  return total;
}
int first_max(const std::vector<double>& vals) {  // max by (value, -rank): lowest rank wins ties
  int best = 0;
  for (int i = 1; i < (int)vals.size(); ++i) if (vals[i] > vals[best]) best = i;
  return best;
}
S rollup(const std::vector<S>& names, const std::vector<int>& ranks,
         const std::vector<std::vector<double>>& cols) {
  Obj avg, med, worst;
  for (size_t k = 0; k < names.size(); ++k) {
    const std::vector<double>& v = cols[k];
    if (v.empty()) {
      avg.kv(names[k], JNULL);
      const S none = Obj().kv("value", JNULL).kv("idx", JNULL).done();
      med.kv(names[k], none); worst.kv(names[k], none);
      continue;
    }
    avg.kv(names[k], jnum(py_sum(v) / (double)v.size()));
    const int mi = closest_to_median(ranks, v), wi = first_max(v);
    med.kv(names[k], Obj().kv("value", jnum(v[mi])).kv("idx", jq(jint(ranks[mi]))).done());
    worst.kv(names[k], Obj().kv("value", jnum(v[wi])).kv("idx", jq(jint(ranks[wi]))).done());
  }
  return Obj().kv("average", avg.done()).kv("median", med.done()).kv("worst", worst.done()).done();
}

tml_trend_in trend_in(const tml_kind_result& k, int series, bool layout_ok) {
  tml_trend_in t;
  memset(&t, 0, sizeof(t));
  if (!k.has_bands || !layout_ok) return t;
  const uint64_t* c = k.band_cnt[series];
  if (c[0] == 0 || c[1] == 0 || c[2] == 0) return t;
  t.valid = 1;
  t.baseline_avg = k.band_sum[series][0] / (double)c[0];
  t.mid_avg = k.band_sum[series][1] / (double)c[1];
  t.recent_avg = k.band_sum[series][2] / (double)c[2];
  return t;
}
// does trend_layout(n, min_points, warmup) exist?  (reduce.py:trend_layout / core.py:51-84)
bool layout_exists(unsigned long long n, unsigned long long min_points, double warmup) {
  if (n < min_points) return false;
  const unsigned long long length = n < 10000 ? n : 10000;
  if (length < min_points) return false;
  const unsigned long long warm = (unsigned long long)std::floor((double)length * warmup);
  return length - warm >= min_points;
}

int run_diag(int (*fn)(const void*, char*, size_t), const void* in, S* out) {
  thread_local std::vector<char> buf;  // reused: no 64 KB zero-fill per rule engine per summary
  if (buf.size() < (1u << 16)) buf.resize(1u << 16);
  int rc = fn(in, buf.data(), buf.size());
  if (rc == TML_ERR_SMALL) { buf.resize(1u << 20); rc = fn(in, buf.data(), buf.size()); }
  if (rc != TML_OK) return rc;
  out->assign(buf.data());
  return TML_OK;
}

enum { S_DL, S_FWD, S_BWD, S_OPT, S_STEP, S_WAIT, S_ALLOC, S_RESV };

}  // namespace

extern "C" int tml_sections_json(const tml_reduce_run_out* o, const tml_sections_args* a, char* json_out,
                                 size_t cap) {
  tml_json::Scope json_scope;
  if (!o || !a || !json_out) return TML_ERR_ARG;
  const int R = (int)o->n_ranks;
  if (R < 1 || R > (int)TML_MAX_RANKS) return TML_ERR_ARG;
  const long long window = (long long)a->window;

  // ranks that hold rows at all; latest observed step
  bool any = false;
  unsigned long long latest = 0;
  int seen = 0;
  for (int r = 0; r < R; ++r)
    if (o->infos[r].n_retained > 0) {
      any = true; ++seen;
      if (o->infos[r].latest_step > latest) latest = o->infos[r].latest_step;
    }
  const S j_latest = any ? jint((long long)latest) : JNULL;
  const S j_training = jint(any ? (long long)latest + 1 : 0);

  // ================================================================ step time
  S step_time;
  {
    const tml_kind_result& k = o->time;
    Obj per_rank, aligned_o;
    for (int r = 0; r < R; ++r)
      if (o->infos[r].t_count > 0)
        per_rank.kv(jint(r), summary_json(summary_from_sums(r, o->infos[r].t_count, o->infos[r].t_sums)));
    std::vector<RankSummary> al;
    for (unsigned i = 0; i < k.n_used; ++i) al.push_back(summary_from_sums(k.used[i], k.n_rows[i], k.t_sums[i]));
    for (const RankSummary& s : al) aligned_o.kv(jint(s.rank), summary_json(s));
    const bool has = !al.empty();
    S win = Obj().kv("alignment", jq("common_steps")).kv("steps_analyzed", jint(has ? (long long)k.n_common : 0))
                .kv("start_step", has ? jint((long long)k.start_step) : JNULL)
                .kv("end_step", has ? jint((long long)k.end_step) : JNULL)
                .kv("window_size", jint(window)).kv("global_ranks_used", jint((long long)al.size()))
                .kv("global_ranks_observed", jint(k.observed)).done();
    S data = Obj().kv("training_steps", j_training).kv("latest_step_observed", j_latest)
                 .kv("aligned_summary", aligned_o.done()).kv("aligned_window", win)
                 .kv("per_global_rank_summary", per_rank.done()).kv("max_rows", jint(window)).done();
    // diagnosis
    tml_st_diag_in din;
    memset(&din, 0, sizeof(din));
    din.n_ranks = (int)al.size();
    din.max_rows = (int)window;
    din.n_common = has ? (long long)k.n_common : 0;
    din.completed_step = has ? (long long)k.end_step : 0;
    for (size_t i = 0; i < al.size(); ++i) {
      tml_rank_means& m = din.ranks[i];
      m.rank = al[i].rank; m.steps_analyzed = al[i].n;
      m.dataloader_ms = al[i].dl; m.forward_ms = al[i].fwd; m.backward_ms = al[i].bwd;
      m.optimizer_ms = al[i].opt; m.step_cpu_ms = al[i].step_cpu;
    }
    const int which = al.size() <= 1 ? 1 : 0;  // single rank -> worst series (trend.py:46)
    const bool lay = layout_exists(k.n_common, 200, 0.10);
    din.trend_step = trend_in(k, S_STEP * 2 + which, lay);
    din.trend_wait = trend_in(k, S_WAIT * 2 + which, lay);
    din.trend_dl = trend_in(k, S_DL * 2 + which, lay);
    S diag;
    int rc = run_diag((int (*)(const void*, char*, size_t))tml_diag_step_time, &din, &diag);
    if (rc != TML_OK) return rc;
    // rollups over the aligned summaries
    std::vector<int> ranks;
    std::vector<std::vector<double>> cols(7);
    for (const RankSummary& s : al) {
      ranks.push_back(s.rank);
      cols[0].push_back(s.total); cols[1].push_back(s.dl); cols[2].push_back(s.compute);
      cols[3].push_back(std::max(0.0, s.traced - ((s.fwd + s.bwd) + s.opt)));
      cols[4].push_back(s.fwd); cols[5].push_back(s.bwd); cols[6].push_back(s.opt);
    }
    const std::vector<S> names = {"total_step_ms", "dataloader_ms", "compute_ms", "wait_ms",
                                  "forward_ms", "backward_ms", "optimizer_ms"};
    S overview;
    if (al.empty()) {
      overview = Obj().kv("rank_comparison", jq("no_data")).kv("median_global_rank", JNULL)
                     .kv("worst_global_rank", JNULL).kv("median_avg_step_ms", JNULL)
                     .kv("worst_avg_step_ms", JNULL).kv("step_time_skew_percent", JNULL).done();
    } else {
      const int wi = first_max(cols[0]), mi = closest_to_median(ranks, cols[0]);
      const double w = cols[0][wi], m = cols[0][mi];
      const bool skew = m > 0.0 && wi != mi;
      overview = Obj().kv("rank_comparison", jq(al.size() <= 1 ? "single_rank" : "distributed"))
                     .kv("median_global_rank", jint(ranks[mi])).kv("worst_global_rank", jint(ranks[wi]))
                     .kv("median_avg_step_ms", jnum(m)).kv("worst_avg_step_ms", jnum(w))
                     .kv("step_time_skew_percent", skew ? jnum(100.0 * (w - m) / m) : JNULL).done();
    }
    step_time = Obj().kv("data", data).kv("diagnosis", diag).kv("global", rollup(names, ranks, cols))
                    .kv("overview", overview).done();
  }

  // ================================================================ process aggregates -> gpu_total
  bool have_gpu_total = false, saw_proc = false, any_gpu_avail = false;
  double gpu_total = 0.0;
  for (int r = 0; r < R; ++r) {
    const tml_proc_agg& p = o->procs[r];
    if (p.n_gpu > 0) { if (!have_gpu_total || p.max_total > gpu_total) gpu_total = p.max_total; have_gpu_total = true; }
    if (p.n > 0) { saw_proc = true; any_gpu_avail = any_gpu_avail || p.any_gpu_available != 0; }
  }
  const bool no_gpu = saw_proc && !any_gpu_avail;

  // ================================================================ step memory
  S step_memory;
  {
    const tml_kind_result& k = o->mem;
    const long long n = k.n_used ? (long long)k.n_common : 0;
    Obj means;
    std::vector<int> ranks;
    std::vector<std::vector<double>> cols(2);
    if (n)
      for (unsigned i = 0; i < k.n_used; ++i) {
        const double ma = k.m_sums[i][0] / (double)n, mr = k.m_sums[i][1] / (double)n;
        means.kv(jint(k.used[i]), Obj().kv("peak_allocated_bytes", jnum(ma)).kv("peak_reserved_bytes", jnum(mr)).done());
        ranks.push_back(k.used[i]);
        if (std::isfinite(ma)) cols[0].push_back(ma);
        if (std::isfinite(mr)) cols[1].push_back(mr);
      }
    tml_mem_diag_in din;
    memset(&din, 0, sizeof(din));
    din.steps_used = n;
    din.window_size = (int)window;
    din.completed_step = k.n_used ? (long long)k.end_step : 0;
    din.ranks_seen = seen;
    din.gpu_total_bytes = (have_gpu_total && gpu_total != 0.0) ? gpu_total : 0.0;
    din.n_metrics = n ? 2 : 0;
    const bool lay = layout_exists(k.n_common, 50, 0.0);
    const int series_of[2][2] = {{S_ALLOC * 2, S_ALLOC * 2 + 1}, {S_RESV * 2, S_RESV * 2 + 1}};
    S metrics = "[";
    for (int mi = 0; mi < din.n_metrics; ++mi) {
      tml_mem_metric_in& m = din.metric[mi];
      m.n_ranks = (int)k.n_used;
      std::vector<double> peaks;
      for (unsigned i = 0; i < k.n_used; ++i) {
        m.ranks[i] = k.used[i];
        m.rank_peak[i] = k.m_sums[i][2 + mi];
        peaks.push_back(k.m_sums[i][2 + mi]);
      }
      m.trend_median = trend_in(k, series_of[mi][0], lay);
      m.trend_worst = trend_in(k, series_of[mi][1], lay);
      m.points = n;
      m.tail_first = k.has_bands ? k.tail_first[series_of[mi][1]] : NAN;
      m.tail_last = k.has_bands ? k.tail_last[series_of[mi][1]] : NAN;
      // the metric's summary as the rule engine derives it (step_memory/model.py:141-221)
      const double med = median_of(peaks);
      const int wi = first_max(peaks);
      const double worst = peaks[wi];
      const double worst_peak = std::max(0.0, worst), median_peak = std::max(0.0, med);
      const double skew_ratio = med > 0.0 ? std::max(0.0, worst / med) : 0.0;
      const double skew_pct = med > 0.0 ? std::max(0.0, (worst - med) / med) : 0.0;
      if (mi) metrics += ",";
      metrics += Obj().kv("metric", jq(mi == 0 ? "peak_allocated" : "peak_reserved"))
          .kv("summary", Obj().kv("window_size", jint(window)).kv("steps_used", jint(n))
                             .kv("median_peak", jnum(median_peak)).kv("worst_peak", jnum(worst_peak))
                             .kv("worst_rank", jint(k.used[wi])).kv("skew_ratio", jnum(skew_ratio))
                             .kv("skew_pct", jnum(skew_pct)).done())
          .kv("coverage", Obj().kv("expected_steps", jint(window)).kv("steps_used", jint(n))
                              .kv("completed_step", k.n_used ? jint((long long)k.end_step) : JNULL)
                              .kv("world_size", jint(seen)).kv("ranks_present", jint(k.n_used))
                              .kv("incomplete", (int)k.n_used < seen ? "true" : "false").done())
          .done();
    }
    metrics += "]";
    S diag;
    int rc = run_diag((int (*)(const void*, char*, size_t))tml_diag_step_memory, &din, &diag);
    if (rc != TML_OK) return rc;
    // step_memory_global: each column only over finite values, keyed by rank string
    std::vector<S> names = {"peak_allocated_bytes", "peak_reserved_bytes"};
    std::vector<std::vector<double>> gcols(2);
    std::vector<int> granks = ranks;
    if (n) { gcols = cols; }
    S global;
    if (n && cols[0].size() == ranks.size() && cols[1].size() == ranks.size()) {
      global = rollup(names, granks, gcols);
    } else {  // empty (or non-finite means: cannot happen with finite byte counts)
      global = rollup(names, std::vector<int>(), std::vector<std::vector<double>>(2));
    }
    step_memory = Obj().kv("training_steps", j_training).kv("latest_step_observed", j_latest)
        .kv("gpu_total_bytes", have_gpu_total ? jnum(gpu_total) : JNULL)
        .kv("no_gpu_detected", no_gpu ? "true" : "false")
        .kv("window", Obj().kv("steps_first", n ? jint((long long)k.start_step) : JNULL)
                          .kv("steps_last", n ? jint((long long)k.end_step) : JNULL).kv("n_steps", jint(n))
                          .kv("window_size", jint(window)).kv("global_ranks_seen", jint(seen))
                          .kv("global_ranks_used", jint(k.n_used)).done())
        .kv("metrics", metrics).kv("per_global_rank", means.done()).kv("diagnosis", diag)
        .kv("global", global).done();
  }

  // ================================================================ process
  S process;
  {
    tml_proc_diag_in din;
    memset(&din, 0, sizeof(din));
    din.n_ranks = a->proc_rows ? R : 0;
    for (int r = 0; r < R; ++r) {
      din.ranks[r] = r;
      din.agg[r] = o->procs[r];
      din.ram_total[r] = a->ram_total;
      din.gpu_count[r] = a->gpu_count;
    }
    int rc = run_diag((int (*)(const void*, char*, size_t))tml_diag_process, &din, &process);
    if (rc != TML_OK) return rc;
  }

  const S all = Obj().kv("step_time", step_time).kv("step_memory", step_memory).kv("process", process).done();
  if (cap < all.size() + 1) return TML_ERR_SMALL;
  memcpy(json_out, all.c_str(), all.size() + 1);
  return TML_OK;
}
