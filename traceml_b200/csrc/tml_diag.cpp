// tml_diag.cpp -- host-side rule engines of libtraceml_b200.so.
//
// O(R) scalar work on the outputs of the window-reduce kernels: rank-level
// median / worst / skew, scores, shares, thresholds, issue ordering and the
// primary diagnosis.  Results leave as one UTF-8 JSON object whose keys mirror
// the reference's DiagnosticResult dataclasses, so the kept payload builders
// (reporting/sections/*/builder.py) can consume them unchanged.
//
// Reference behaviour implemented here (paths under src/traceml/):
//   step time   diagnostics/step_time/adapters.py:142-355, context.py:84-532,
//               rules.py:87-296, api.py:118-649, trend.py:36-147, policy.py:55-73
//   step memory reporting/sections/step_memory/model.py:130-219,
//               diagnostics/step_memory/adapters.py:72-172, rules.py:96-283,
//               api.py:284-508, trend.py:203-277, policy.py:12-36
//   process     reporting/sections/process/loader.py:56-230,
//               diagnostics/process/context.py:140-340, rules.py:57-345,
//               api.py:52-118, policy.py:21-31, diagnostics/bands.py:21-34

#include <ctype.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include <charconv>

#include "../../include/traceml_b200.h"
#include "tml_internal.h"

namespace {

// ------------------------------------------------------------------ JSON helpers
typedef tml_json::Str S;  // arena-backed: see tml_internal.h

S fmt(const char* f, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, f);
  vsnprintf(buf, sizeof(buf), f, ap);
  va_end(ap);
  return S(buf);
}

S jstr(const S& s) {
  bool plain = true;
  for (unsigned char ch : s) if (ch == '"' || ch == '\\' || ch < 0x20) { plain = false; break; }
  if (plain) { S o; o.reserve(s.size() + 2); o += '"'; o += s; o += '"'; return o; }
  S o = "\"";
  for (unsigned char ch : s) {
    if (ch == '"') o += "\\\"";
    else if (ch == '\\') o += "\\\\";
    else if (ch == '\n') o += "\\n";
    else if (ch < 0x20) o += fmt("\\u%04x", ch);
    else o += (char)ch;
  }
  return o + "\"";
}
S jnum(double v) {
  if (!isfinite(v)) return "null";
  char buf[40];  // shortest text that round-trips the double exactly (what Python's repr prints)
  char* end = std::to_chars(buf, buf + 36, v).ptr;
  bool is_float = false;
  for (const char* p = buf; p < end; ++p) if (*p == '.' || *p == 'e' || *p == 'E' || *p == 'n') { is_float = true; break; }
  if (!is_float) { *end++ = '.'; *end++ = '0'; }  // keep it a JSON float
  return S(buf, end);
}
S jint(long long v) {
  char buf[24];
  return S(buf, std::to_chars(buf, buf + sizeof(buf), v).ptr);
}
S jbool(bool b) { return b ? "true" : "false"; }
const S JNULL = "null";
S jopt_int(long long v, bool has) { return has ? jint(v) : JNULL; }
S jopt_num(double v, bool has) { return has ? jnum(v) : JNULL; }

struct Obj {
  S s;
  bool first = true;
  Obj() { s.reserve(240); s += '{'; }  // one allocation for the typical object
  Obj& kv(const char* k, const S& v) {  // keys are identifiers: no escaping needed
    if (!first) s += ',';
    first = false;
    s += '"'; s += k; s += "\":"; s += v;
    return *this;
  }
  S done() { s += '}'; return std::move(s); }  // the object is spent afterwards
};
S jarr(const std::vector<S>& v) {
  S o = "[";
  for (size_t i = 0; i < v.size(); ++i) { if (i) o += ","; o += v[i]; }
  return o + "]";
}

int emit(const S& s, char* out, size_t cap) {
  if (!out || cap < s.size() + 1) return TML_ERR_SMALL;
  memcpy(out, s.c_str(), s.size() + 1);
  return TML_OK;
}

// ------------------------------------------------------------------ scalars
inline double ffin(double v) { return isfinite(v) ? v : 0.0; }          // model.py:31-34
inline double nnf(double v) { return isfinite(v) ? (v > 0.0 ? v : 0.0) : 0.0; }  // context.py:84-95
inline double share(double v, double total) {                           // context.py:98-105
  double t = nnf(total);
  if (t <= 0.0) return 0.0;
  double q = nnf(v) / t;
  return q > 0.0 ? q : 0.0;
}
S pct1(double v) { return fmt("%.1f%%", nnf(v) * 100.0); }
S rank_s(int r) { return r >= 0 ? fmt("r%d", r) : S("\xe2\x80\x94"); }  // em dash

double median_of(std::vector<double> v) {  // numpy.median / model.py:130-138
  if (v.empty()) return 0.0;
  std::sort(v.begin(), v.end());
  size_t n = v.size(), m = n / 2;
  return (n & 1) ? v[m] : (v[m - 1] + v[m]) / 2.0;
}

struct Issue {
  S kind, status, severity, summary, action, metric, phase;
  bool has_metric = false, has_phase = false;
  bool has_score = false, has_share = false, has_skew = false;
  double score = 0, share_pct = 0, skew_pct = 0;
  std::vector<int> ranks;
  S evidence = "{}";
  S json() const {
    std::vector<S> rk;
    for (int r : ranks) rk.push_back(jint(r));
    return Obj().kv("kind", jstr(kind)).kv("status", jstr(status)).kv("severity", jstr(severity))
        .kv("summary", jstr(summary)).kv("action", jstr(action))
        .kv("metric", has_metric ? jstr(metric) : JNULL).kv("phase", has_phase ? jstr(phase) : JNULL)
        .kv("score", jopt_num(score, has_score)).kv("share_pct", jopt_num(share_pct, has_share))
        .kv("skew_pct", jopt_num(skew_pct, has_skew)).kv("ranks", jarr(rk)).kv("evidence", evidence)
        .done();
  }
};
int sev_rank(const S& s) { return s == "crit" ? 2 : (s == "warn" ? 1 : 0); }

// ================================================================== step time
struct Thresholds {  // policy.py:55-73 (summary policy)
  double in_str_warn = 0.10, in_str_crit = 0.18, cp_str_warn = 0.10, cp_str_crit = 0.18;
  double in_share_warn = 0.30, in_share_crit = 0.40, wait_warn = 0.18, wait_crit = 0.28;
  double in_bound_max_skew = 0.05, cp_bound_max_skew = 0.05;
  double cp_share_warn = 0.88, cp_share_crit = 0.94;
  int min_steps_confident = 20, min_steps_for_diag = 50;
};

struct Metric {
  double median_total = 0, worst_total = 0, skew_ratio = 0, skew_pct = 0;
  int worst_rank = -1;
};

struct StDiag {
  S kind, severity, reason, action, note;
  bool has_note = false;
  long long steps_used = 0;
  int worst_rank = -1;
};
const char* st_status(const S& k) {
  if (k == "NO_DATA") return "NO DATA";
  if (k == "WARMUP") return "WARMUP";
  if (k == "BALANCED") return "BALANCED";
  if (k == "STRAGGLER") return "STRAGGLER";
  if (k == "INPUT_STRAGGLER") return "INPUT STRAGGLER";
  if (k == "COMPUTE_STRAGGLER") return "COMPUTE STRAGGLER";
  if (k == "INPUT_BOUND") return "INPUT-BOUND";
  if (k == "COMPUTE_BOUND") return "COMPUTE-BOUND";
  return "WAIT-HEAVY";
}
int st_priority(const S& k) {  // api.py:65-72
  if (k == "STRAGGLER") return 50;
  if (k == "INPUT_STRAGGLER") return 40;
  if (k == "COMPUTE_STRAGGLER") return 39;
  if (k == "INPUT_BOUND") return 30;
  if (k == "WAIT_HEAVY") return 20;
  if (k == "COMPUTE_BOUND") return 10;
  return 0;
}
S st_diag_json(const StDiag& d) {
  return Obj().kv("severity", jstr(d.severity)).kv("status", jstr(st_status(d.kind)))
      .kv("reason", jstr(d.reason)).kv("action", jstr(d.action)).kv("kind", jstr(d.kind))
      .kv("steps_used", jint(d.steps_used)).kv("worst_rank", jopt_int(d.worst_rank, d.worst_rank >= 0))
      .kv("note", d.has_note ? jstr(d.note) : JNULL).kv("confidence", JNULL).done();
}
S st_result(const StDiag& d, const std::vector<Issue>& issues, const S& attribution) {
  std::vector<S> is;
  for (const Issue& i : issues) is.push_back(i.json());
  return Obj().kv("primary", st_diag_json(d)).kv("issues", jarr(is))
      .kv("metric_attribution", attribution).done();
}
StDiag st_warmup(long long low_in, long long required_in, long long high_in) {  // api.py:118-152
  long long low = std::max(0LL, low_in), high = std::max(low, high_in);
  long long req = std::max(1LL, required_in);
  S avail = (low == high) ? fmt("%lld", low) : fmt("%lld-%lld", low, high);
  StDiag d;
  d.kind = "WARMUP"; d.severity = "info";
  d.reason = "Only " + avail + (high == 1 ? " step" : " steps") +
             " per rank available; summary diagnosis requires " + fmt("%lld", req) + ".";
  d.action = "Use a longer run for a stable timing diagnosis.";
  d.steps_used = low;
  return d;
}

bool trend_pct(const tml_trend_in& t, double* pct) {  // core.py:96-102,118-129
  if (!t.valid) return false;
  if (fabs(t.baseline_avg) <= 1e-12) return false;
  *pct = (t.recent_avg - t.baseline_avg) / t.baseline_avg;
  return true;
}
S trend_fmt(double p, double deadband) {  // core.py:132-146
  if (fabs(p) < deadband) return fmt("~ %+.1f%%", p * 100.0);
  return S(p > 0 ? "\xe2\x86\x91" : "\xe2\x86\x93") + fmt(" %+.1f%%", p * 100.0);
}

struct TopEntry { int rank; double v; };
S top_ranks(const std::vector<int>& ranks, const std::vector<double>& vals) {  // api.py:192-233
  if (ranks.empty()) return "[]";
  std::vector<TopEntry> e;
  for (size_t i = 0; i < ranks.size(); ++i) e.push_back({ranks[i], nnf(vals[i])});
  std::stable_sort(e.begin(), e.end(), [](const TopEntry& a, const TopEntry& b) {
    if (a.v != b.v) return a.v > b.v;
    return a.rank < b.rank;
  });
  std::vector<double> sorted;
  for (auto& x : e) sorted.push_back(x.v);
  std::sort(sorted.begin(), sorted.end());
  double med = sorted[sorted.size() / 2];  // NB upper median
  std::vector<S> out;
  for (size_t i = 0; i < e.size() && i < 3; ++i) {
    double ex = std::max(0.0, e[i].v - med);
    out.push_back(Obj().kv("rank", jint(e[i].rank)).kv("value_ms", jnum(e[i].v))
                      .kv("excess_vs_median_ms", jnum(ex))
                      .kv("pct_vs_median", med > 0.0 ? jnum(ex / med) : JNULL).done());
  }
  return jarr(out);
}

}  // namespace

extern "C" int tml_diag_step_time(const tml_st_diag_in* in, char* json_out, size_t cap) {
  tml_json::Scope json_scope;
  if (!in || in->n_ranks < 0 || in->n_ranks > (int)TML_MAX_RANKS) return TML_ERR_ARG;
  const Thresholds th;
  const int n = in->n_ranks;
  if (n == 0) return emit("null", json_out, cap);  // adapters.py:250-251

  // ranks in ascending id order (adapters.py:253)
  std::vector<int> order(n);
  for (int i = 0; i < n; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(),
                   [&](int a, int b) { return in->ranks[a].rank < in->ranks[b].rank; });
  std::vector<int> ranks(n);
  std::vector<double> dl(n), fw(n), bw(n), op(n), raw(n), comp(n), eff(n), wait(n);
  long long min_steps = 0, max_steps = 0;
  for (int k = 0; k < n; ++k) {
    const tml_rank_means& r = in->ranks[order[k]];
    ranks[k] = r.rank;
    dl[k] = ffin(r.dataloader_ms); fw[k] = ffin(r.forward_ms); bw[k] = ffin(r.backward_ms);
    op[k] = ffin(r.optimizer_ms); raw[k] = ffin(r.step_cpu_ms);
    comp[k] = (fw[k] + bw[k]) + op[k];
    eff[k] = std::max(raw[k], comp[k]);
    wait[k] = std::max(0.0, eff[k] - comp[k]);
    long long s = r.steps_analyzed;
    if (k == 0 || s < min_steps) min_steps = s;
    if (k == 0 || s > max_steps) max_steps = s;
  }
  if (min_steps < th.min_steps_for_diag)  // adapters.py:254-259
    return emit(st_result(st_warmup(min_steps, th.min_steps_for_diag, max_steps), {}, "{}"),
                json_out, cap);

  const long long steps_used = in->n_common > 0 ? in->n_common : min_steps;  // adapters.py:289-291
  const bool single = n <= 1;

  // overall worst rank: max by (dl + eff, -rank)  (adapters.py:311-316)
  int overall_worst = ranks[0];
  {
    double best = dl[0] + eff[0];
    for (int k = 1; k < n; ++k) {
      double s = dl[k] + eff[k];
      if (s > best) { best = s; overall_worst = ranks[k]; }
    }
  }

  // adapters.py:142-197
  auto make_metric = [&](const std::vector<double>& v, int override_rank) {
    Metric m;
    m.median_total = median_of(v);
    int wi = 0;
    for (int k = 1; k < n; ++k) if (v[k] > v[wi]) wi = k;  // np.argmax: first max
    m.worst_total = v[wi];
    m.worst_rank = ranks[wi];
    if (n <= 1) { m.median_total = m.worst_total; m.skew_ratio = 0; m.skew_pct = 0; }
    else if (m.median_total > 0.0) {
      m.skew_ratio = m.worst_total / m.median_total;
      m.skew_pct = (m.worst_total - m.median_total) / m.median_total;
    }
    if (override_rank >= 0) m.worst_rank = override_rank;
    return m;
  };
  const Metric m_dl = make_metric(dl, -1), m_fw = make_metric(fw, -1), m_bw = make_metric(bw, -1);
  const Metric m_op = make_metric(op, -1), m_st = make_metric(eff, overall_worst);
  const Metric m_wt = make_metric(wait, -1);

  auto total_of = [&](const Metric& m) { return nnf(single ? m.worst_total : m.median_total); };
  auto skew_of = [&](const Metric& m) { return single ? 0.0 : nnf(m.skew_pct); };
  const double step_total = total_of(m_st);

  if (step_total <= 0.0) {  // api.py:355-364
    StDiag d;
    d.kind = "NO_DATA"; d.severity = "info"; d.reason = "No usable step-time data yet.";
    d.action = "Wait for the first complete window."; d.steps_used = steps_used;
    d.worst_rank = overall_worst;
    return emit(st_result(d, {}, "{}"), json_out, cap);
  }
  if (steps_used < th.min_steps_confident) {  // api.py:366-373
    StDiag d = st_warmup(steps_used, th.min_steps_confident, steps_used);
    d.worst_rank = overall_worst;
    return emit(st_result(d, {}, "{}"), json_out, cap);
  }

  // ---- context (context.py:393-532)
  const double dl_total = total_of(m_dl), wait_total = total_of(m_wt);
  const double comp_total = total_of(m_fw) + total_of(m_bw) + total_of(m_op);
  struct Cand { const char* label; double share, skew; int worst_rank; };
  std::vector<Cand> cands;
  const Metric* cm[3] = {&m_fw, &m_bw, &m_op};
  const char* cl[3] = {"Forward", "Backward", "Optimizer"};
  for (int i = 0; i < 3; ++i) {
    double t = total_of(*cm[i]);
    if (t <= 0.0) continue;
    cands.push_back({cl[i], share(t, step_total), skew_of(*cm[i]), cm[i]->worst_rank});
  }
  const Cand* dominant = nullptr;  // max by (skew, share), first wins ties
  const Cand* largest = nullptr;   // max by share
  for (const Cand& c : cands) {
    if (!dominant || c.skew > dominant->skew || (c.skew == dominant->skew && c.share > dominant->share))
      dominant = &c;
    if (!largest || c.share > largest->share) largest = &c;
  }
  const double comp_skew = dominant ? dominant->skew : 0.0;
  const int comp_rank = dominant ? dominant->worst_rank : overall_worst;
  const double dl_share = share(dl_total, step_total), wait_share = share(wait_total, step_total);
  const double comp_share = share(comp_total, step_total);
  const double dl_skew = skew_of(m_dl);
  const int dl_rank = m_dl.worst_rank;

  const double med_comp = nnf(m_fw.median_total) + nnf(m_bw.median_total) + nnf(m_op.median_total);
  const double wst_comp = nnf(m_fw.worst_total) + nnf(m_bw.worst_total) + nnf(m_op.worst_total);
  const double typical = nnf(m_dl.median_total) + med_comp;
  double in_score = 0.0, cp_score = 0.0;
  if (typical > 0.0) {
    in_score = std::max(0.0, nnf(m_dl.worst_total) - nnf(m_dl.median_total)) / typical;
    cp_score = std::max(0.0, wst_comp - med_comp) / typical;
  }
  auto sev = [](double v, double crit) { return S(nnf(v) >= crit ? "crit" : "warn"); };
  auto lower = [](const char* s) { S o(s); for (auto& ch : o) ch = (char)tolower(ch); return o; };

  // ---- rules, in registration order (rules.py:277-285)
  std::vector<Issue> issues;
  int idx_in = -1, idx_cp = -1;
  if (!single && in_score >= th.in_str_warn) {
    Issue i;
    i.kind = "INPUT_STRAGGLER"; i.status = "INPUT STRAGGLER"; i.severity = sev(in_score, th.in_str_crit);
    i.summary = rank_s(dl_rank) + " has excess dataloader burden (~" + pct1(in_score) +
                " of a typical local step).";
    i.action = "Inspect input loading on " + rank_s(dl_rank) + ".";
    i.metric = "dataloader_fetch"; i.phase = "dataloader"; i.has_metric = i.has_phase = true;
    i.has_score = i.has_share = i.has_skew = true;
    i.score = nnf(in_score); i.share_pct = nnf(dl_share); i.skew_pct = nnf(dl_skew);
    if (dl_rank >= 0) i.ranks.push_back(dl_rank);
    idx_in = (int)issues.size();
    issues.push_back(i);
  }
  if (!single && cp_score >= th.cp_str_warn) {
    S label = dominant ? lower(dominant->label) : S("compute");
    Issue i;
    i.kind = "COMPUTE_STRAGGLER"; i.status = "COMPUTE STRAGGLER"; i.severity = sev(cp_score, th.cp_str_crit);
    i.summary = rank_s(comp_rank) + " has excess compute burden (~" + pct1(cp_score) +
                " of a typical local step).";
    i.action = "Inspect " + label + " on " + rank_s(comp_rank) + ".";
    i.metric = "compute"; i.phase = label; i.has_metric = i.has_phase = true;
    i.has_score = i.has_share = i.has_skew = true;
    i.score = nnf(cp_score); i.share_pct = nnf(comp_share); i.skew_pct = nnf(comp_skew);
    if (comp_rank >= 0) i.ranks.push_back(comp_rank);
    idx_cp = (int)issues.size();
    issues.push_back(i);
  }
  if (dl_share >= th.in_share_warn && !(!single && dl_skew > th.in_bound_max_skew)) {
    Issue i;
    i.kind = "INPUT_BOUND"; i.status = "INPUT-BOUND"; i.severity = sev(dl_share, th.in_share_crit);
    i.summary = "Dataloader is " + pct1(dl_share) + " of the typical step.";
    i.action = "Increase workers, prefetch, or storage throughput.";
    i.metric = "dataloader_fetch"; i.phase = "dataloader"; i.has_metric = i.has_phase = true;
    i.has_share = i.has_skew = true; i.share_pct = nnf(dl_share); i.skew_pct = nnf(dl_skew);
    if (dl_rank >= 0) i.ranks.push_back(dl_rank);
    issues.push_back(i);
  }
  if (wait_share >= th.wait_warn) {
    Issue i;
    i.kind = "WAIT_HEAVY"; i.status = "WAIT-HEAVY"; i.severity = sev(wait_share, th.wait_crit);
    i.summary = "WAIT* is " + pct1(wait_share) + " of the typical step.";
    i.action = "Inspect work outside traced phases, CPU stalls, logging, checkpointing, "
               "validation, or transfers.";
    i.metric = "wait_proxy"; i.phase = "wait"; i.has_metric = i.has_phase = true;
    i.has_share = true; i.share_pct = nnf(wait_share);
    if (overall_worst >= 0) i.ranks.push_back(overall_worst);
    issues.push_back(i);
  }
  if (comp_share >= th.cp_share_warn && !(dl_share >= th.in_share_warn) &&
      !(wait_share >= th.wait_warn) && !(!single && comp_skew > th.cp_bound_max_skew)) {
    S label = largest ? lower(largest->label) : S("compute");
    Issue i;
    i.kind = "COMPUTE_BOUND"; i.status = "COMPUTE-BOUND"; i.severity = sev(comp_share, th.cp_share_crit);
    i.summary = "Compute-bound; " + label + " is the largest phase.";
    i.action = "Optimize model compute or reduce step cost.";
    i.metric = "compute"; i.phase = label; i.has_metric = i.has_phase = true;
    i.has_share = i.has_skew = true; i.share_pct = nnf(comp_share); i.skew_pct = nnf(comp_skew);
    if (overall_worst >= 0) i.ranks.push_back(overall_worst);
    issues.push_back(i);
  }
  const bool both = idx_in >= 0 && idx_cp >= 0;
  const S in_sev = idx_in >= 0 ? issues[idx_in].severity : S();
  const S in_sum = idx_in >= 0 ? issues[idx_in].summary : S();
  const S in_act = idx_in >= 0 ? issues[idx_in].action : S();
  const S cp_sev = idx_cp >= 0 ? issues[idx_cp].severity : S();
  const S cp_sum = idx_cp >= 0 ? issues[idx_cp].summary : S();
  const S cp_act = idx_cp >= 0 ? issues[idx_cp].action : S();
  const double max_score = std::max(in_score, cp_score);
  const double max_crit = std::max(th.in_str_crit, th.cp_str_crit);
  if (both) {  // api.py:387-434
    Issue i;
    i.kind = "STRAGGLER"; i.status = "STRAGGLER"; i.severity = sev(max_score, max_crit);
    i.summary = "Both input and compute are uneven across ranks.";
    i.action = "Inspect the slowest rank and both dominant phases.";
    i.metric = "step_time"; i.phase = "combined"; i.has_metric = i.has_phase = true;
    i.has_score = true; i.score = max_score;
    std::vector<int> rs;
    if (dl_rank >= 0) rs.push_back(dl_rank);
    if (comp_rank >= 0 && comp_rank != dl_rank) rs.push_back(comp_rank);
    std::sort(rs.begin(), rs.end());
    i.ranks = rs;
    i.evidence = Obj().kv("input_score", jnum(in_score)).kv("compute_score", jnum(cp_score)).done();
    issues.push_back(i);
  }
  // diagnostics/common.py:105-121: sorted(..., reverse=True) is stable w.r.t. the
  // reversed input, i.e. equal keys keep their ORIGINAL relative order.
  std::stable_sort(issues.begin(), issues.end(), [](const Issue& a, const Issue& b) {
    int sa = sev_rank(a.severity), sb = sev_rank(b.severity);
    if (sa != sb) return sa > sb;
    double ca = a.has_score ? a.score : 0.0, cb = b.has_score ? b.score : 0.0;
    if (ca != cb) return ca > cb;
    return a.ranks.size() > b.ranks.size();
  });
  const Issue* top = nullptr;  // api.py:263-279
  for (const Issue& i : issues) {
    if (!top) { top = &i; continue; }
    int pa = st_priority(i.kind), pb = st_priority(top->kind);
    double ca = i.has_score ? i.score : 0.0, cb = top->has_score ? top->score : 0.0;
    if (pa > pb || (pa == pb && ca > cb)) top = &i;
  }

  StDiag d;
  d.steps_used = steps_used;
  auto multi = [&](int r) { return single ? -1 : r; };
  if (both) {
    d.kind = "STRAGGLER"; d.severity = sev(max_score, max_crit);
    d.reason = "Both input and compute are uneven across ranks.";
    d.action = "Inspect the slowest rank and both dominant phases.";
    d.worst_rank = in_score >= cp_score ? dl_rank : comp_rank;
    d.has_note = true;
    d.note = "Input score " + pct1(in_score) + ", compute score " + pct1(cp_score) + ".";
  } else if (idx_in >= 0) {
    d.kind = "INPUT_STRAGGLER"; d.severity = in_sev; d.reason = in_sum; d.action = in_act;
    d.worst_rank = dl_rank; d.has_note = true;
    d.note = "Dataloader share is " + pct1(dl_share) + ".";
  } else if (idx_cp >= 0) {
    d.kind = "COMPUTE_STRAGGLER"; d.severity = cp_sev; d.reason = cp_sum; d.action = cp_act;
    d.worst_rank = comp_rank; d.has_note = true;
    d.note = "Compute share is " + pct1(comp_share) + ".";
  } else if (top && top->kind == "INPUT_BOUND") {
    d.kind = "INPUT_BOUND"; d.severity = top->severity; d.reason = top->summary; d.action = top->action;
    d.worst_rank = multi(dl_rank);
  } else if (top && top->kind == "WAIT_HEAVY") {
    d.kind = "WAIT_HEAVY"; d.severity = top->severity; d.reason = top->summary; d.action = top->action;
    d.worst_rank = multi(overall_worst); d.has_note = true;
    d.note = "wait_ms = total_step_ms - dataloader_ms - compute_ms.";
  } else if (top && top->kind == "COMPUTE_BOUND") {
    d.kind = "COMPUTE_BOUND"; d.severity = top->severity; d.reason = top->summary; d.action = top->action;
    d.worst_rank = multi(overall_worst);
  } else {
    d.kind = "BALANCED"; d.severity = "info";
    d.reason = "No dominant bottleneck is visible in this window.";
    d.action = "Focus on throughput only if overall speed is still low.";
    d.worst_rank = multi(overall_worst);
  }

  // ---- trend note (trend.py:67-147): min 100 steps, +-8 % gates, 3 % dead-band
  if (steps_used >= 100 && in->n_common > 0) {
    double ps = 0, pw = 0, pd = 0;
    const bool hs = trend_pct(in->trend_step, &ps), hw = trend_pct(in->trend_wait, &pw);
    const bool hd = trend_pct(in->trend_dl, &pd);
    auto state = [](bool has, double p) -> const char* {
      if (!has) return nullptr;
      if (p >= 0.08) return "worsening";
      if (p <= -0.08) return "improving";
      return nullptr;
    };
    const char *ss = state(hs, ps), *ws = state(hw, pw), *ds = state(hd, pd);
    S tn;
    if ((d.kind == "INPUT_BOUND" || d.kind == "INPUT_STRAGGLER") && ds)
      tn = S("Trend: dataloader is ") + ds + " (" + trend_fmt(pd, 0.03) + ").";
    else if ((d.kind == "COMPUTE_BOUND" || d.kind == "COMPUTE_STRAGGLER" || d.kind == "STRAGGLER") && ss)
      tn = S("Trend: step time is ") + ss + " (" + trend_fmt(ps, 0.03) + ").";
    else if (d.kind == "WAIT_HEAVY" && ws)
      tn = S("Trend: WAIT* is ") + ws + " (" + trend_fmt(pw, 0.03) + ").";
    else if (d.kind == "BALANCED" && ss && S(ss) == "worsening" &&
             (wait_share >= th.wait_warn * 0.90 || dl_share >= th.in_share_warn * 0.90))
      tn = "Trend: step time is rising (" + trend_fmt(ps, 0.03) + ").";
    if (!tn.empty()) {
      d.note = d.has_note ? (d.note + " " + tn) : tn;
      d.has_note = true;
    }
  }

  if (issues.empty()) {  // api.py:541-556
    Issue i;
    i.kind = d.kind; i.status = st_status(d.kind); i.severity = d.severity;
    i.summary = d.reason; i.action = d.action;
    if (d.worst_rank >= 0) i.ranks.push_back(d.worst_rank);
    issues.push_back(i);
  }

  // ---- metric attribution (api.py:236-260,558-641)
  auto attr = [&](const Metric& m, const char* key, const char* phase, const std::vector<double>& rv) {
    return Obj().kv("metric", jstr(key)).kv("phase", jstr(phase))
        .kv("median_total_ms", jnum(nnf(m.median_total))).kv("worst_total_ms", jnum(nnf(m.worst_total)))
        .kv("worst_rank", jopt_int(m.worst_rank, m.worst_rank >= 0)).kv("skew_pct", jnum(skew_of(m)))
        .kv("share_pct", jnum(share(total_of(m), step_total))).kv("top_ranks", top_ranks(ranks, rv))
        .done();
  };
  std::vector<double> comp_rv(n);
  for (int k = 0; k < n; ++k) comp_rv[k] = (nnf(fw[k]) + nnf(bw[k])) + nnf(op[k]);
  S compute_attr = Obj().kv("metric", jstr("compute"))
      .kv("phase", jstr(dominant ? lower(dominant->label) : S("compute")))
      .kv("median_total_ms", jnum(med_comp)).kv("worst_total_ms", jnum(wst_comp))
      .kv("worst_rank", jopt_int(comp_rank, comp_rank >= 0)).kv("skew_pct", jnum(comp_skew))
      .kv("share_pct", jnum(comp_share)).kv("top_ranks", top_ranks(ranks, comp_rv)).done();
  S attribution = Obj()
      .kv("dataloader_fetch", attr(m_dl, "dataloader_fetch", "dataloader", dl))
      .kv("forward", attr(m_fw, "forward", "forward", fw))
      .kv("backward", attr(m_bw, "backward", "backward", bw))
      .kv("optimizer_step", attr(m_op, "optimizer_step", "optimizer", op))
      .kv("wait_proxy", attr(m_wt, "wait_proxy", "wait", wait))
      .kv("step_time", attr(m_st, "step_time", "step", eff))
      .kv("compute", compute_attr).done();
  return emit(st_result(d, issues, attribution), json_out, cap);
}

// ================================================================== step memory
namespace {

struct MemTh {  // policy.py:12-36
  int min_steps = 50;
  double p_warn = 0.92, p_crit = 0.97, k_warn = 0.12, k_crit = 0.20;
  double score_scale = 100.0 * 1024.0 * 1024.0, confirmed_delta = 1024.0 * 1024.0 * 1024.0;
};

struct Creep {
  bool eligible = false, early = false, confirmed = false;
  double base = 0, mid = 0, recent = 0, abs_delta = 0, score = 0;
  bool has_wg = false, has_mg = false;
  double wg = 0, mg = 0;
};

struct MemSig {
  S metric;
  long long steps_used = 0;
  int window_size = 0;
  long long completed_step = 0;
  int ranks_seen = 0, worst_rank = -1;
  double worst_peak = 0, median_peak = 0, skew_ratio = 0, skew_pct = 0;
  bool has_pressure = false;
  double pressure = 0;
  Creep creep;
};

S mem_label(const S& m) { S o = m; for (auto& c : o) if (c == '_') c = ' '; return o; }
const char* mem_status(const S& k) {
  if (k == "NO_DATA") return "NO DATA";
  if (k == "BALANCED") return "BALANCED";
  if (k == "HIGH_PRESSURE") return "HIGH PRESSURE";
  if (k == "IMBALANCE") return "IMBALANCE";
  if (k == "CREEP_EARLY") return "MEMORY RISING";
  return "MEMORY CREEP";
}
int mem_prio(const S& k) {
  if (k == "HIGH_PRESSURE") return 0;
  if (k == "IMBALANCE") return 1;
  if (k == "CREEP_CONFIRMED") return 2;
  if (k == "CREEP_EARLY") return 3;
  return 100;
}
S creep_note(const Creep& c) {  // rules.py:37-57
  S o = fmt("baseline %.0f B -> recent %.0f B", c.base, c.recent);
  o += fmt(", %s%.0f B", c.abs_delta >= 0.0 ? "+" : "-", fabs(c.abs_delta));
  if (c.has_wg) o += fmt(", (~%.0f%%)", c.wg * 100.0);
  return o;
}
S mem_diag(const S& kind, const S& sev, const S& metric, long long steps, const S& reason,
           const S& action, int worst_rank, const S* note, double conf, bool has_conf) {
  return Obj().kv("severity", jstr(sev)).kv("status", jstr(mem_status(kind))).kv("reason", jstr(reason))
      .kv("action", jstr(action)).kv("kind", jstr(kind)).kv("metric", jstr(metric))
      .kv("steps_used", jint(steps)).kv("worst_rank", jopt_int(worst_rank, worst_rank >= 0))
      .kv("note", note ? jstr(*note) : JNULL).kv("confidence", jopt_num(conf, has_conf)).done();
}

}  // namespace

extern "C" int tml_diag_step_memory(const tml_mem_diag_in* in, char* json_out, size_t cap) {
  tml_json::Scope json_scope;
  if (!in || in->n_metrics < 0 || in->n_metrics > 2) return TML_ERR_ARG;
  const MemTh th;
  const char* names[2] = {"peak_allocated", "peak_reserved"};
  std::vector<MemSig> sigs;
  std::vector<Issue> issues;
  for (int mi = 0; mi < in->n_metrics; ++mi) {
    const tml_mem_metric_in& m = in->metric[mi];
    if (m.n_ranks <= 0 || m.n_ranks > (int)TML_MAX_RANKS) return TML_ERR_ARG;
    MemSig s;
    s.metric = names[mi];
    s.steps_used = in->steps_used; s.window_size = in->window_size;
    s.completed_step = in->completed_step; s.ranks_seen = m.n_ranks;
    // rank order ascending (model.py:146)
    std::vector<int> order(m.n_ranks);
    for (int i = 0; i < m.n_ranks; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return m.ranks[a] < m.ranks[b]; });
    std::vector<double> peaks;
    for (int i : order) peaks.push_back(m.rank_peak[i]);
    double med = median_of(peaks);
    int wi = 0;
    for (int k = 1; k < m.n_ranks; ++k) if (peaks[k] > peaks[wi]) wi = k;  // list.index(max): first
    double worst = peaks[wi];
    s.worst_rank = m.ranks[order[wi]];
    s.worst_peak = std::max(0.0, worst); s.median_peak = std::max(0.0, med);
    s.skew_ratio = med > 0.0 ? std::max(0.0, worst / med) : 0.0;
    s.skew_pct = med > 0.0 ? std::max(0.0, (worst - med) / med) : 0.0;
    if (in->gpu_total_bytes > 0.0) {
      s.has_pressure = true;
      s.pressure = std::max(0.0, s.worst_peak / in->gpu_total_bytes);
    }
    // window creep (trend.py:203-277)
    Creep& c = s.creep;
    if (s.steps_used >= th.min_steps && m.trend_worst.valid && m.trend_median.valid) {
      const tml_trend_in &w = m.trend_worst, &d = m.trend_median;
      c.eligible = true;
      c.base = w.baseline_avg; c.mid = w.mid_avg; c.recent = w.recent_avg;
      c.abs_delta = w.recent_avg - w.baseline_avg;
      if (fabs(w.baseline_avg) > 1e-12) { c.has_wg = true; c.wg = c.abs_delta / w.baseline_avg; }
      if (fabs(d.baseline_avg) > 1e-12) {
        c.has_mg = true; c.mg = (d.recent_avg - d.baseline_avg) / d.baseline_avg;
      }
      const bool recent_gt_mid = (w.recent_avg - w.mid_avg) > 0.0 && (d.recent_avg - d.mid_avg) > 0.0;
      const bool mid_gt_base = (w.mid_avg > w.baseline_avg) && (d.mid_avg > d.baseline_avg);
      const bool ok = recent_gt_mid && mid_gt_base;
      c.early = ok && c.abs_delta > 0.0;
      c.confirmed = ok && c.abs_delta >= th.confirmed_delta;
      c.score = std::max(0.0, c.abs_delta) / std::max(1.0, th.score_scale) +
                std::max(0.0, c.has_wg ? c.wg : 0.0) * 10.0 + std::max(0.0, c.has_mg ? c.mg : 0.0) * 6.0;
    }
    // rules (rules.py:96-224), per metric, then sorted
    std::vector<Issue> local;
    auto mk = [&](const char* kind, const char* status, const S& sev, const S& summary,
                  const char* action, double score, const S& evidence) {
      Issue i;
      i.kind = kind; i.status = status; i.severity = sev; i.summary = summary; i.action = action;
      i.metric = s.metric; i.phase = "memory"; i.has_metric = i.has_phase = true;
      i.has_score = true; i.score = score; i.has_skew = true; i.skew_pct = s.skew_pct;
      if (s.worst_rank >= 0) i.ranks.push_back(s.worst_rank);
      i.evidence = evidence;
      local.push_back(i);
    };
    const bool ready = s.steps_used >= th.min_steps;
    if (s.has_pressure && ready && s.pressure >= th.p_warn)
      mk("HIGH_PRESSURE", "HIGH PRESSURE", s.pressure >= th.p_crit ? "crit" : "warn",
         mem_label(s.metric) + fmt(" is near device capacity (~%.0f%%).", s.pressure * 100.0),
         "Reduce memory load.", s.pressure, Obj().kv("pressure_frac", jnum(s.pressure)).done());
    if (ready && !(s.skew_pct < th.k_warn))
      mk("IMBALANCE", "IMBALANCE", s.skew_pct >= th.k_crit ? "crit" : "warn",
         mem_label(s.metric) + fmt(" shows +%.1f%% cross-rank skew.", s.skew_pct * 100.0),
         "Inspect per-rank workload.", s.skew_pct, Obj().kv("skew_pct", jnum(s.skew_pct)).done());
    if (c.confirmed || c.early) {
      S ev = Obj().kv("overall_abs_delta_bytes", jnum(c.abs_delta))
                 .kv("overall_worst_growth_pct", jopt_num(c.wg, c.has_wg))
                 .kv("overall_median_growth_pct", jopt_num(c.mg, c.has_mg))
                 .kv("note", jstr(creep_note(c))).done();
      if (c.confirmed)
        mk("CREEP_CONFIRMED", "MEMORY CREEP", "warn",
           mem_label(s.metric) + " is rising across the window.", "Check retained tensors or caches.",
           c.score, ev);
      else
        mk("CREEP_EARLY", "MEMORY RISING", "info",
           mem_label(s.metric) + " is rising from early to recent steps.", "Watch the next window.",
           c.score, ev);
    }
    for (auto& i : local) issues.push_back(i);
    sigs.push_back(s);
  }
  // rules.py:235-254
  std::stable_sort(issues.begin(), issues.end(), [](const Issue& a, const Issue& b) {
    int pa = mem_prio(a.kind), pb = mem_prio(b.kind);
    if (pa != pb) return pa < pb;
    int sa = sev_rank(a.severity), sb = sev_rank(b.severity);
    if (sa != sb) return sa > sb;
    if (a.score != b.score) return a.score > b.score;
    return a.metric < b.metric;
  });

  auto sig_json = [&](const MemSig& s) {
    const Creep& c = s.creep;
    S trend = Obj().kv("eligible", jbool(c.eligible))
        .kv("baseline_avg_bytes", jopt_num(c.base, c.eligible)).kv("mid_avg_bytes", jopt_num(c.mid, c.eligible))
        .kv("recent_avg_bytes", jopt_num(c.recent, c.eligible))
        .kv("overall_abs_delta_bytes", jopt_num(c.abs_delta, c.eligible))
        .kv("overall_worst_growth_pct", jopt_num(c.wg, c.eligible && c.has_wg))
        .kv("overall_median_growth_pct", jopt_num(c.mg, c.eligible && c.has_mg))
        .kv("early", jbool(c.early)).kv("confirmed", jbool(c.confirmed)).kv("score", jnum(c.score)).done();
    return Obj().kv("metric", jstr(s.metric)).kv("device", JNULL).kv("steps_used", jint(s.steps_used))
        .kv("window_size", jint(s.window_size)).kv("completed_step", jint(s.completed_step))
        .kv("ranks_seen", jint(s.ranks_seen)).kv("worst_rank", jopt_int(s.worst_rank, s.worst_rank >= 0))
        .kv("worst_peak_bytes", jnum(s.worst_peak)).kv("median_peak_bytes", jnum(s.median_peak))
        .kv("skew_ratio", jnum(s.skew_ratio)).kv("skew_pct", jnum(s.skew_pct))
        .kv("pressure_frac", jopt_num(s.pressure, s.has_pressure)).kv("trend", trend).done();
  };
  Obj attribution;
  for (const MemSig& s : sigs) attribution.kv(s.metric.c_str(), sig_json(s));

  S primary;
  if (!issues.empty()) {  // api.py:396-433
    const Issue& t = issues[0];
    const MemSig* sg = nullptr;
    for (const MemSig& s : sigs) if (s.metric == t.metric) sg = &s;
    double conf = 0;
    bool has_conf = true;
    if (t.kind == "HIGH_PRESSURE") conf = t.severity == "crit" ? 0.9 : 0.8;
    else if (t.kind == "IMBALANCE") conf = t.severity == "crit" ? 0.85 : 0.75;
    else if (t.kind == "CREEP_CONFIRMED") conf = 0.88;
    else if (t.kind == "CREEP_EARLY") conf = 0.60;
    else has_conf = false;
    S note;
    const S* np = nullptr;
    if ((t.kind == "CREEP_CONFIRMED" || t.kind == "CREEP_EARLY") && sg) { note = creep_note(sg->creep); np = &note; }
    int wr = !t.ranks.empty() ? t.ranks[0] : (sg ? sg->worst_rank : -1);
    primary = mem_diag(t.kind, t.severity, t.metric, sg ? sg->steps_used : 0, t.summary, t.action, wr,
                       np, conf, has_conf);
  } else if (sigs.empty()) {  // api.py:444-453
    primary = mem_diag("NO_DATA", "info", "peak_reserved", 0, "No step-memory data yet.",
                       "Wait for more completed steps.", -1, nullptr, 0.0, true);
  } else {  // api.py:463-497
    std::vector<const MemSig*> ready;
    for (const MemSig& s : sigs) if (s.steps_used >= th.min_steps) ready.push_back(&s);
    if (ready.empty()) {
      const MemSig* best = &sigs[0];
      for (const MemSig& s : sigs) if (s.steps_used > best->steps_used) best = &s;
      primary = mem_diag("NO_DATA", "info", best->metric, best->steps_used,
                         fmt("Need at least %d completed steps.", th.min_steps), "Keep monitoring.",
                         best->worst_rank, nullptr, 0.0, true);
    } else {
      const MemSig* base = nullptr;
      for (const MemSig* s : ready) if (s->metric == "peak_reserved") base = s;
      if (!base) for (const MemSig* s : ready) if (s->metric == "peak_allocated") base = s;
      if (!base) base = ready[0];
      primary = mem_diag("BALANCED", "info", base->metric, base->steps_used,
                         "No clear pressure, imbalance, or creep signal.", "Keep monitoring.",
                         base->worst_rank, nullptr, 0.75, true);
    }
  }
  std::vector<S> is;
  for (const Issue& i : issues) is.push_back(i.json());
  return emit(Obj().kv("primary", primary).kv("issues", jarr(is))
                  .kv("metric_attribution", attribution.done()).done(),
              json_out, cap);
}

// ================================================================== process
namespace {

const char* band_of(bool has, double v, double low_below, bool has_low, double high_at, bool has_high,
                    double very_high_at, bool has_vh) {  // bands.py:21-34
  if (!has) return "";
  if (has_vh && v >= very_high_at) return "very_high";
  if (has_high && v >= high_at) return "high";
  if (has_low && v < low_below) return "low";
  return "normal";
}

struct RankAgg {
  int rank;
  bool has_gpu;
  double cpu_avg, cpu_peak, ram_avg, ram_peak, ram_total;
  double used_avg, used_peak, resv_avg, resv_peak, total, ratio;
  bool has_ratio;
  int cores, gpu_count;
  bool gpu_available;
  uint64_t n;
};

}  // namespace

extern "C" int tml_diag_process(const tml_proc_diag_in* in, char* json_out, size_t cap) {
  tml_json::Scope json_scope;
  if (!in || in->n_ranks < 0 || in->n_ranks > (int)TML_MAX_RANKS) return TML_ERR_ARG;
  std::vector<RankAgg> rs;
  std::vector<int> order(in->n_ranks);
  for (int i = 0; i < in->n_ranks; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return in->ranks[a] < in->ranks[b]; });
  // pooled aggregates (loader.py:56-139): AVG = sum / count over all rows of all ranks
  // The byte sums pool as exact integers (64 ranks of u64 sums fit in 128 bits) and round once
  // per average, as the reference's exact integer AVG does; a double accumulator rounds as soon
  // as the pooled total passes 2^53.
  uint64_t n_all = 0, n_gpu_all = 0;
  double s_cpu = 0, s_cpu_lo = 0;
  unsigned __int128 s_rss = 0, s_used = 0, s_resv = 0;
  auto dd_add = [](double& hi, double& lo, double xh, double xl) {  // TwoSum accumulate
    const double s = hi + xh, bp = s - hi;
    const double err = (hi - (s - bp)) + (xh - bp);
    hi = s; lo = (lo + xl) + err;
  };
  double mx_cpu = -INFINITY, mx_rss = -INFINITY, mx_used = -INFINITY, mx_resv = -INFINITY;
  double mx_total = -INFINITY, mx_ramtot = -INFINITY, ts_min = INFINITY, ts_max = -INFINITY;
  int mx_cores = -1, mx_gpucount = -1, any_avail = -1, distinct = 0;
  for (int oi : order) {
    const tml_proc_agg& a = in->agg[oi];
    if (a.n == 0) continue;
    ++distinct;
    RankAgg r;
    r.rank = in->ranks[oi]; r.n = a.n; r.has_gpu = a.n_gpu > 0;
    r.cpu_avg = (a.sum_cpu + a.sum_cpu_lo) / (double)a.n; r.cpu_peak = a.max_cpu;
    r.ram_avg = a.sum_rss / (double)a.n; r.ram_peak = a.max_rss; r.ram_total = in->ram_total[oi];
    r.used_avg = r.has_gpu ? a.sum_used / (double)a.n_gpu : 0; r.used_peak = a.max_used;
    r.resv_avg = r.has_gpu ? a.sum_resv / (double)a.n_gpu : 0; r.resv_peak = a.max_resv;
    r.total = a.max_total; r.has_ratio = a.max_ratio >= 0.0; r.ratio = a.max_ratio;
    r.cores = (int)a.max_cores; r.gpu_available = a.any_gpu_available != 0;
    r.gpu_count = r.gpu_available ? in->gpu_count[oi] : 0;
    rs.push_back(r);
    n_all += a.n; n_gpu_all += a.n_gpu;
    dd_add(s_cpu, s_cpu_lo, a.sum_cpu, a.sum_cpu_lo);
    s_rss += a.sum_rss; s_used += a.sum_used; s_resv += a.sum_resv;
    mx_cpu = std::max(mx_cpu, a.max_cpu); mx_rss = std::max(mx_rss, a.max_rss);
    if (r.has_gpu) {
      mx_used = std::max(mx_used, a.max_used); mx_resv = std::max(mx_resv, a.max_resv);
      mx_total = std::max(mx_total, a.max_total);
    }
    mx_ramtot = std::max(mx_ramtot, r.ram_total);
    ts_min = std::min(ts_min, a.ts_min); ts_max = std::max(ts_max, a.ts_max);
    mx_cores = std::max(mx_cores, r.cores); mx_gpucount = std::max(mx_gpucount, r.gpu_count);
    any_avail = std::max(any_avail, r.gpu_available ? 1 : 0);
  }
  const bool have = n_all > 0, have_gpu = n_gpu_all > 0;
  const double cpu_avg = have ? (s_cpu + s_cpu_lo) / (double)n_all : 0;
  // (double) of an unsigned __int128 rounds to nearest, like Python's float(int)
  const double ram_avg = have ? (double)s_rss / (double)n_all : 0;
  const double used_avg = have_gpu ? (double)s_used / (double)n_gpu_all : 0;
  const double resv_avg = have_gpu ? (double)s_resv / (double)n_gpu_all : 0;

  // ---- signals (context.py:242-340)
  auto frac = [](bool hn, double num, bool hd, double den, double* out) {
    if (!hn || !hd || den <= 0.0) return false;
    *out = std::max(0.0, num / den);
    return true;
  };
  double cpu_cap = 0, ram_pct = 0, used_pct = 0, resv_pct = 0;
  const bool h_cpu = have && mx_cores > 0;
  if (h_cpu) cpu_cap = std::max(0.0, cpu_avg / (100.0 * (double)mx_cores)) * 100.0;
  bool h_ram = frac(have, mx_rss, have, mx_ramtot, &ram_pct);
  bool h_used = frac(have_gpu, mx_used, have_gpu, mx_total, &used_pct);
  bool h_resv = frac(have_gpu, mx_resv, have_gpu, mx_total, &resv_pct);
  ram_pct *= 100.0; used_pct *= 100.0; resv_pct *= 100.0;

  auto best_rank = [&](auto getter, auto has) {  // first strict max in rank order
    int best = -1; double bv = 0;
    for (const RankAgg& r : rs) { if (!has(r)) continue; double v = getter(r); if (best < 0 || v > bv) { best = r.rank; bv = v; } }
    return best;
  };
  auto imbalance = [&](auto getter, auto has, double* out) {
    double mx = -INFINITY, mn = INFINITY; int cnt = 0;
    for (const RankAgg& r : rs) { if (!has(r)) continue; double v = getter(r); mx = std::max(mx, v); mn = std::min(mn, v); ++cnt; }
    if (cnt < 2) return false;
    *out = mx <= 0.0 ? 0.0 : std::max(0.0, (mx - mn) / mx);
    return true;
  };
  auto any = [](const RankAgg&) { return true; };
  auto gpu = [](const RankAgg& r) { return r.has_gpu; };
  const int hi_rss = best_rank([](const RankAgg& r) { return r.ram_peak; }, any);
  const int hi_used = best_rank([](const RankAgg& r) { return r.used_peak; }, gpu);
  const int hi_resv = best_rank([](const RankAgg& r) { return r.resv_peak; }, gpu);
  int lh_rank = -1; double lh_bytes = 0;
  for (const RankAgg& r : rs) {
    if (!r.has_gpu) continue;
    double head = std::max(r.total - r.resv_peak, 0.0);
    if (lh_rank < 0 || head < lh_bytes) { lh_rank = r.rank; lh_bytes = head; }
  }
  int oh_rank = -1; double oh_ratio = 0;
  for (const RankAgg& r : rs) {
    double ratio; bool hr = r.has_ratio;
    if (hr) ratio = r.ratio;
    else hr = frac(r.has_gpu, r.resv_peak, r.has_gpu, r.used_peak, &ratio);
    if (!hr) continue;
    if (oh_rank < 0 || ratio > oh_ratio) { oh_rank = r.rank; oh_ratio = ratio; }
  }
  double used_imb = 0, resv_imb = 0;
  const bool h_uimb = imbalance([](const RankAgg& r) { return r.used_peak; }, gpu, &used_imb);
  const bool h_rimb = imbalance([](const RankAgg& r) { return r.resv_peak; }, gpu, &resv_imb);
  used_imb *= 100.0; resv_imb *= 100.0;

  // ---- rules (rules.py:71-294)
  std::vector<Issue> issues;
  if (have) {
    const bool use_resv = h_resv;
    const bool hp = use_resv ? h_resv : h_used;
    const double pct = use_resv ? resv_pct : used_pct;
    const char* metric = use_resv ? "gpu_mem_reserved_peak_percent" : "gpu_mem_used_peak_percent";
    const int rank = use_resv ? hi_resv : hi_used;
    S band = band_of(hp, pct, 30.0, true, 80.0, true, 90.0, true);
    S on_rank = rank >= 0 ? fmt(" on rank %d", rank) : S();
    S ev = Obj().kv("gpu_mem_used_peak_percent", jopt_num(used_pct, h_used))
               .kv("gpu_mem_reserved_peak_percent", jopt_num(resv_pct, h_resv))
               .kv("rank", jopt_int(rank, rank >= 0)).done();
    auto mk = [&](const char* kind, const char* sev, const S& summary, const char* action,
                  const char* mname, const char* phase, double score, std::vector<int> ranks, const S& evd) {
      Issue i;
      i.kind = kind; i.status = kind;
      for (auto& ch : i.status) if (ch == '_') ch = ' ';
      i.severity = sev; i.summary = summary; i.action = action; i.metric = mname; i.phase = phase;
      i.has_metric = i.has_phase = true; i.has_score = true; i.score = score; i.ranks = ranks;
      i.evidence = evd;
      issues.push_back(i);
    };
    std::vector<int> rk; if (rank >= 0) rk.push_back(rank);
    if (band == "very_high")
      mk("VERY_HIGH_PROCESS_GPU_MEMORY", "crit",
         fmt("Process GPU memory was very high, peaking at %.1f%%", pct) + on_rank + ".",
         "Reduce traced process GPU memory pressure.", metric, "gpu_memory", pct, rk, ev);
    if (band == "high")
      mk("HIGH_PROCESS_GPU_MEMORY", "warn",
         fmt("Process GPU memory was high, peaking at %.1f%%", pct) + on_rank + ".",
         "Watch traced process GPU memory headroom.", metric, "gpu_memory", pct, rk, ev);
    if (oh_rank >= 0 && oh_ratio >= 1.5) {
      std::vector<int> r1{oh_rank};
      mk("GPU_MEMORY_RESERVED_OVERHANG", "warn", fmt("Reserved GPU memory was %.2fx active use.", oh_ratio),
         "Inspect allocator behavior or retained tensors.", "gpu_mem_reserved_peak_bytes", "gpu_memory",
         oh_ratio, r1,
         Obj().kv("gpu_mem_reserved_overhang_ratio", jnum(oh_ratio)).kv("highest_overhang_rank", jint(oh_rank)).done());
    }
    {
      bool hi = h_rimb; double ip = resv_imb; const char* im = "rank_gpu_reserved_imbalance_percent";
      std::vector<int> ir;
      if (hi_resv >= 0) ir.push_back(hi_resv);
      if (lh_rank >= 0) ir.push_back(lh_rank);
      if (!hi) {
        hi = h_uimb; ip = used_imb; im = "rank_gpu_used_imbalance_percent";
        ir.clear();
        if (hi_used >= 0) ir.push_back(hi_used);
        if (lh_rank >= 0) ir.push_back(lh_rank);
      }
      if (hi && ip >= 30.0)
        mk("RANK_GPU_MEMORY_IMBALANCE", "warn", fmt("Process GPU memory differed by %.1f%% across ranks.", ip),
           "Inspect per-rank workload and memory behavior.", im, "gpu_memory", ip, ir,
           Obj().kv("rank_gpu_used_imbalance_percent", jopt_num(used_imb, h_uimb))
               .kv("rank_gpu_reserved_imbalance_percent", jopt_num(resv_imb, h_rimb))
               .kv("highest_used_rank", jopt_int(hi_used, hi_used >= 0))
               .kv("highest_reserved_rank", jopt_int(hi_resv, hi_resv >= 0))
               .kv("least_headroom_rank", jopt_int(lh_rank, lh_rank >= 0)).done());
    }
    if (h_ram && S(band_of(true, ram_pct, 30.0, true, 80.0, true, 0, false)) == "high") {
      std::vector<int> r1; if (hi_rss >= 0) r1.push_back(hi_rss);
      mk("HIGH_PROCESS_RSS", "warn", fmt("Process RSS was high, peaking at %.1f%%.", ram_pct),
         "Reduce traced process host memory pressure.", "ram_peak_percent", "ram", ram_pct, r1,
         Obj().kv("ram_peak_percent", jnum(ram_pct)).kv("highest_rss_rank", jopt_int(hi_rss, hi_rss >= 0)).done());
    }
    if (h_cpu && S(band_of(true, cpu_cap, 30.0, true, 80.0, true, 0, false)) == "high")
      mk("HIGH_PROCESS_CPU", "warn", fmt("Process CPU averaged %.1f%% of capacity.", cpu_cap),
         "Inspect data loading, preprocessing, or host contention.", "cpu_capacity_percent", "cpu", cpu_cap, {},
         Obj().kv("cpu_avg_percent", jnum(cpu_avg)).kv("cpu_logical_core_count", jint(mx_cores))
             .kv("cpu_capacity_percent", jnum(cpu_cap)).done());
    auto prio = [](const S& k) {
      if (k == "VERY_HIGH_PROCESS_GPU_MEMORY") return 0;
      if (k == "HIGH_PROCESS_GPU_MEMORY") return 1;
      if (k == "GPU_MEMORY_RESERVED_OVERHANG") return 2;
      if (k == "RANK_GPU_MEMORY_IMBALANCE") return 3;
      if (k == "HIGH_PROCESS_RSS") return 4;
      return 5;
    };
    std::stable_sort(issues.begin(), issues.end(), [&](const Issue& a, const Issue& b) {
      int pa = prio(a.kind), pb = prio(b.kind);
      if (pa != pb) return pa < pb;
      return a.score > b.score;
    });
  }

  S primary;
  auto pd = [&](const S& kind, const S& sev, const S& status, const S& reason, const S& action) {
    return Obj().kv("severity", jstr(sev)).kv("status", jstr(status)).kv("reason", jstr(reason))
        .kv("action", jstr(action)).kv("kind", jstr(kind)).kv("samples_used", jint((long long)n_all)).done();
  };
  if (!issues.empty()) {
    const Issue& t = issues[0];
    primary = pd(t.kind, t.severity, t.status, t.summary, t.action);
  } else if (!have) {
    primary = pd("NO_DATA", "info", "NO DATA", "No traced process telemetry was recorded.",
                 "Collect process telemetry for workload-local context.");
  } else {
    primary = pd("NORMAL", "info", "NORMAL",
                 (h_used || h_resv) ? "Process CPU, RSS, and GPU memory showed no pressure."
                                    : "Process CPU and RSS showed no pressure.",
                 "Use training diagnostics for model-level bottlenecks.");
  }

  S agg = Obj().kv("first_ts", jopt_num(ts_min, have)).kv("last_ts", jopt_num(ts_max, have))
      .kv("process_samples", jint((long long)n_all)).kv("distinct_global_ranks", jint(distinct))
      .kv("cpu_avg_percent", jopt_num(cpu_avg, have)).kv("cpu_peak_percent", jopt_num(mx_cpu, have))
      .kv("cpu_logical_core_count", jopt_int(mx_cores, have && mx_cores >= 0))
      .kv("ram_avg_bytes", jopt_num(ram_avg, have)).kv("ram_peak_bytes", jopt_num(mx_rss, have))
      .kv("ram_total_bytes", jopt_num(mx_ramtot, have))
      .kv("gpu_available", have ? jbool(any_avail > 0) : JNULL)
      .kv("gpu_count", jopt_int(mx_gpucount, have && mx_gpucount >= 0))
      .kv("gpu_mem_used_avg_bytes", jopt_num(used_avg, have_gpu)).kv("gpu_mem_used_peak_bytes", jopt_num(mx_used, have_gpu))
      .kv("gpu_mem_reserved_avg_bytes", jopt_num(resv_avg, have_gpu))
      .kv("gpu_mem_reserved_peak_bytes", jopt_num(mx_resv, have_gpu))
      .kv("gpu_mem_total_bytes", jopt_num(mx_total, have_gpu)).done();
  Obj per_rank;
  for (const RankAgg& r : rs) {
    per_rank.kv(fmt("%d", r.rank).c_str(),
        Obj().kv("global_rank", jint(r.rank)).kv("cpu_avg_percent", jnum(r.cpu_avg))
            .kv("cpu_peak_percent", jnum(r.cpu_peak)).kv("cpu_logical_core_count", jint(r.cores))
            .kv("ram_avg_bytes", jnum(r.ram_avg)).kv("ram_peak_bytes", jnum(r.ram_peak))
            .kv("ram_total_bytes", jnum(r.ram_total)).kv("gpu_available", jbool(r.gpu_available))
            .kv("gpu_count", jint(r.gpu_count))
            .kv("gpu_mem_used_avg_bytes", jopt_num(r.used_avg, r.has_gpu))
            .kv("gpu_mem_used_peak_bytes", jopt_num(r.used_peak, r.has_gpu))
            .kv("gpu_mem_reserved_avg_bytes", jopt_num(r.resv_avg, r.has_gpu))
            .kv("gpu_mem_reserved_peak_bytes", jopt_num(r.resv_peak, r.has_gpu))
            .kv("gpu_mem_total_bytes", jopt_num(r.total, r.has_gpu))
            .kv("gpu_mem_reserved_overhang_ratio", jopt_num(r.ratio, r.has_ratio)).done());
  }
  std::vector<S> is;
  for (const Issue& i : issues) is.push_back(i.json());
  return emit(Obj().kv("primary", primary).kv("issues", jarr(is)).kv("aggregate", agg)
                  .kv("per_global_rank", per_rank.done()).done(),
              json_out, cap);
}

// ================================================================== system
namespace {

// One node's issues (context.py:285-373, rules.py:55-310, policy.py:22-36) in DEFAULT_SYSTEM_RULES
// order, each scoped to the node (api.py:106-170) with samples_used = the node's samples.
void sys_node_issues(const tml_sys_diag_in* in, std::vector<Issue>& issues) {
  const tml_sys_agg& a = in->agg;
  const bool have = a.n > 0, hg = a.n_gpu > 0;
  const int n_gpus = have ? (int)std::min<uint32_t>(a.n_gpus, TML_SYS_MAX_GPUS) : 0;
  char label_buf[33];
  memcpy(label_buf, in->node_label, 32);
  label_buf[32] = 0;
  const S label(label_buf);
  const bool has_node_rank = in->node_rank >= 0;

  // ---- node signals (context.py:285-373); every GPU index < n_gpus has all its values
  auto frac = [](double num, double den, double* out) {  // context.py:154-164
    if (den <= 0.0) return false;
    *out = std::max(0.0, num / den);
    return true;
  };
  double ram_pct = 0.0;
  const bool h_ram = have && frac(a.ram_peak, a.ram_total, &ram_pct);
  if (h_ram) ram_pct = ram_pct * 100.0;
  double mem_frac = 0.0, pow_frac = 0.0;
  int hi_mem_idx = -1, hi_pow_idx = -1, hi_temp_idx = -1, lo_util_idx = -1;
  double best_mem = 0.0, best_pow = 0.0, best_temp = 0.0, best_util = 0.0;
  bool h_mem = false, h_pow = false;
  for (int g = 0; g < n_gpus; ++g) {
    const tml_sys_gpu_agg& q = a.gpu[g];
    double f;
    if (frac(q.mem_peak, q.mem_total, &f)) {
      if (!h_mem || f > mem_frac) mem_frac = f;
      if (hi_mem_idx < 0 || f > best_mem) { hi_mem_idx = g; best_mem = f; }
      h_mem = true;
    }
    if (frac(q.power_avg, q.power_limit, &f)) {
      if (!h_pow || f > pow_frac) pow_frac = f;
      if (hi_pow_idx < 0 || f > best_pow) { hi_pow_idx = g; best_pow = f; }
      h_pow = true;
    }
    if (hi_temp_idx < 0 || q.temp_peak > best_temp) { hi_temp_idx = g; best_temp = q.temp_peak; }
    if (lo_util_idx < 0 || q.util_avg < best_util) { lo_util_idx = g; best_util = q.util_avg; }
  }
  const double mem_pct = mem_frac * 100.0, pow_pct = pow_frac * 100.0;

  // ---- rules, in DEFAULT_SYSTEM_RULES order; SYSTEM_ISSUE_PRIORITY is that same order
  auto pct_s = [](double v) { return fmt("%.1f%%", v); };  // rules.py:13-14
  auto mk = [&](const char* kind, const char* status, const char* sev, S summary, const char* action,
                const char* metric, const char* phase, double score, int gpu, const S& ev_head) {
    Issue i;
    i.kind = kind; i.status = status; i.severity = sev; i.action = action;
    i.metric = metric; i.phase = phase; i.has_metric = i.has_phase = true;
    i.has_score = true; i.score = score;
    if (gpu >= 0) i.ranks.push_back(gpu);
    // _scoped_issue / _scope_text (api.py:106-150)
    Obj scope;
    scope.kv("level", jstr(gpu >= 0 ? "gpu" : "node")).kv("node", jstr(label))
        .kv("node_rank", jopt_int(in->node_rank, has_node_rank));
    if (gpu >= 0) {
      scope.kv("gpu_idx", jint(gpu));
      const S existing = fmt(" on gpu%d", gpu), suffix = S(" on ") + label + fmt(" gpu%d", gpu);
      const size_t at = summary.find(existing);
      if (at != S::npos) {
        S o;
        size_t from = 0, p = at;
        while (p != S::npos) { o += summary.substr(from, p - from); o += suffix; from = p + existing.size(); p = summary.find(existing, from); }
        o += summary.substr(from);
        summary = o;
      } else {
        while (!summary.empty() && summary.back() == '.') summary.pop_back();
        summary += suffix + ".";
      }
    } else if (!label.empty()) {
      while (!summary.empty() && summary.back() == '.') summary.pop_back();
      summary += S(" on ") + label + ".";
    }
    i.summary = summary;
    S ev = ev_head;  // the rule's evidence, then scope and samples_used
    ev.pop_back();
    if (ev.size() > 1) ev += ",";
    ev += "\"scope\":"; ev += scope.done();
    ev += ",\"samples_used\":"; ev += jint((long long)a.n);
    ev += "}";
    i.evidence = ev;
    issues.push_back(i);
  };
  auto gpu_suffix = [](int g) { return g >= 0 ? fmt(" on gpu%d", g) : S(); };
  if (have) {
    const S mem_band = band_of(h_mem, mem_pct, 30.0, true, 80.0, true, 90.0, true);
    const S mem_ev = Obj().kv("gpu_mem_peak_percent", jopt_num(mem_pct, h_mem))
                         .kv("gpu_idx", jopt_int(hi_mem_idx, hi_mem_idx >= 0)).done();
    if (mem_band == "very_high")
      mk("VERY_HIGH_GPU_MEMORY", "VERY HIGH GPU MEMORY", "crit",
         S("GPU memory was very high, peaking at ") + pct_s(mem_pct) + gpu_suffix(hi_mem_idx) + ".",
         "Reduce GPU memory pressure before scaling this run.", "gpu_mem_peak_percent", "gpu_memory", mem_pct,
         hi_mem_idx, mem_ev);
    if (S(band_of(hg, a.gpu_temp_peak, 0, false, 85.0, true, 0, false)) == "high")
      mk("HIGH_GPU_TEMPERATURE", "HIGH GPU TEMPERATURE", "crit",
         fmt("GPU temperature was high, peaking at %.1f C", a.gpu_temp_peak) + gpu_suffix(hi_temp_idx) + ".",
         "Check cooling and thermal throttling risk.", "gpu_temp_peak_c", "gpu_temperature", a.gpu_temp_peak,
         hi_temp_idx,
         Obj().kv("gpu_temp_peak_c", jnum(a.gpu_temp_peak)).kv("gpu_idx", jopt_int(hi_temp_idx, hi_temp_idx >= 0)).done());
    if (mem_band == "high")
      mk("HIGH_GPU_MEMORY", "HIGH GPU MEMORY", "warn",
         S("GPU memory was high, peaking at ") + pct_s(mem_pct) + gpu_suffix(hi_mem_idx) + ".",
         "Watch GPU memory headroom for larger batches or models.", "gpu_mem_peak_percent", "gpu_memory", mem_pct,
         hi_mem_idx, mem_ev);
    if (S(band_of(h_pow, pow_pct, 30.0, true, 80.0, true, 0, false)) == "high")
      mk("HIGH_GPU_POWER", "HIGH GPU POWER", "warn",
         S("GPU power was high, averaging ") + pct_s(pow_pct) + " of limit" + gpu_suffix(hi_pow_idx) + ".",
         "Review power headroom if this run is unstable.", "gpu_power_avg_limit_percent", "gpu_power", pow_pct,
         hi_pow_idx,
         Obj().kv("gpu_power_avg_limit_percent", jnum(pow_pct)).kv("gpu_idx", jopt_int(hi_pow_idx, hi_pow_idx >= 0)).done());
    if (S(band_of(h_ram, ram_pct, 30.0, true, 80.0, true, 0, false)) == "high")
      mk("HIGH_HOST_MEMORY", "HIGH HOST MEMORY", "warn",
         S("Host RAM usage was high, peaking at ") + pct_s(ram_pct) + " of total.",
         "Reduce host memory pressure or inspect data workers.", "ram_peak_percent", "ram", ram_pct, -1,
         Obj().kv("ram_peak_percent", jnum(ram_pct)).done());
    if (S(band_of(true, a.cpu_avg, 30.0, true, 80.0, true, 0, false)) == "high")
      mk("HIGH_CPU", "HIGH CPU", "warn", S("CPU usage was high, averaging ") + pct_s(a.cpu_avg) + ".",
         "Inspect CPU-side preprocessing or host contention.", "cpu_avg_percent", "cpu", a.cpu_avg, -1,
         Obj().kv("cpu_avg_percent", jnum(a.cpu_avg)).done());
    if (S(band_of(hg, a.gpu_util_avg, 30.0, true, 80.0, true, 0, false)) == "low")
      mk("LOW_GPU_UTILIZATION", "LOW GPU UTILIZATION", "info",
         S("GPU utilization was low, averaging ") + pct_s(a.gpu_util_avg) + ".",
         "Use step-time diagnostics to check host or input stalls.", "gpu_util_avg_percent", "gpu_utilization",
         100.0 - a.gpu_util_avg, lo_util_idx,
         Obj().kv("gpu_util_avg_percent", jnum(a.gpu_util_avg))
             .kv("lowest_util_gpu_idx", jopt_int(lo_util_idx, lo_util_idx >= 0)).done());
  }
}

// The diagnosis primary (api.py:68-103, 173-186): the first issue, scoped, with the samples of its
// node; without one, the default from the cluster aggregate `a`.
S sys_primary(const std::vector<Issue>& issues, long long issue_samples, const tml_sys_agg& a) {
  const bool have = a.n > 0, hg = a.n_gpu > 0;
  auto pd = [&](const S& kind, const S& sev, const S& status, const S& reason, const S& action, long long used,
                const S& scope) {
    return Obj().kv("severity", jstr(sev)).kv("status", jstr(status)).kv("reason", jstr(reason))
        .kv("action", jstr(action)).kv("kind", jstr(kind)).kv("samples_used", jint(used)).kv("scope", scope).done();
  };
  S primary;
  if (!issues.empty()) {
    const Issue& t = issues[0];
    const size_t at = t.evidence.find("\"scope\":");
    const size_t end = t.evidence.find('}', at);
    primary = pd(t.kind, t.severity, t.status, t.summary, t.action, issue_samples,
                 t.evidence.substr(at + 8, end + 1 - (at + 8)));
  } else if (!have) {
    primary = pd("NO_DATA", "info", "NO DATA", "No system telemetry was recorded.",
                 "Collect system telemetry for host-level context.", 0, Obj().kv("level", jstr("cluster")).done());
  } else {
    // cluster signals carry no per-GPU rows: only the utilisation / temperature columns count
    primary = pd("NORMAL", "info", "NORMAL",
                 hg ? "CPU, RAM, and GPU showed no system pressure." : "CPU and RAM showed no system pressure.",
                 "Use training diagnostics for model-level bottlenecks.", (long long)a.n,
                 Obj().kv("level", jstr("cluster")).done());
  }
  return primary;
}

// SystemSummaryAgg (model.py:50-81, loader.py:97-125) of `a`.
S sys_agg_json(const tml_sys_agg& a) {
  const bool have = a.n > 0, hg = a.n_gpu > 0;
  return Obj().kv("first_ts", jopt_num(a.first_ts, have)).kv("last_ts", jopt_num(a.last_ts, have))
      .kv("system_samples", jint((long long)a.n))
      .kv("cpu_avg_percent", jopt_num(a.cpu_avg, have)).kv("cpu_peak_percent", jopt_num(a.cpu_peak, have))
      .kv("ram_avg_bytes", jopt_num(a.ram_avg, have)).kv("ram_peak_bytes", jopt_num(a.ram_peak, have))
      .kv("ram_total_bytes", jopt_num(a.ram_total, have))
      .kv("gpu_available", have ? jbool(a.gpu_available != 0) : JNULL)
      .kv("gpu_count", jopt_int(a.gpu_count, have))
      .kv("gpu_util_avg_percent", jopt_num(a.gpu_util_avg, hg)).kv("gpu_util_peak_percent", jopt_num(a.gpu_util_peak, hg))
      .kv("gpu_mem_avg_bytes", jopt_num(a.gpu_mem_avg, hg)).kv("gpu_mem_peak_bytes", jopt_num(a.gpu_mem_peak, hg))
      .kv("gpu_temp_avg_c", jopt_num(a.gpu_temp_avg, hg)).kv("gpu_temp_peak_c", jopt_num(a.gpu_temp_peak, hg))
      .kv("gpu_power_avg_w", jopt_num(a.gpu_power_avg, hg)).kv("gpu_power_peak_w", jopt_num(a.gpu_power_peak, hg))
      .done();
}

// The PerGPUSummary rows (model.py:84-117, loader.py:128-156) of a node's aggregates.
S sys_per_gpu_json(const tml_sys_agg& a) {
  const int n_gpus = a.n > 0 ? (int)std::min<uint32_t>(a.n_gpus, TML_SYS_MAX_GPUS) : 0;
  Obj per_gpu;
  for (int g = 0; g < n_gpus; ++g) {
    const tml_sys_gpu_agg& q = a.gpu[g];
    per_gpu.kv(fmt("%d", g).c_str(),
        Obj().kv("gpu_idx", jint(g)).kv("util_avg_percent", jnum(q.util_avg)).kv("util_peak_percent", jnum(q.util_peak))
            .kv("mem_avg_bytes", jnum(q.mem_avg)).kv("mem_peak_bytes", jnum(q.mem_peak))
            .kv("mem_total_bytes", jnum(q.mem_total)).kv("temp_avg_c", jnum(q.temp_avg))
            .kv("temp_peak_c", jnum(q.temp_peak)).kv("power_avg_w", jnum(q.power_avg))
            .kv("power_peak_w", jnum(q.power_peak)).kv("power_limit_w", jnum(q.power_limit)).done());
  }
  return per_gpu.done();
}

int sys_priority(const S& kind) {  // SYSTEM_ISSUE_PRIORITY (rules.py:273-281)
  static const char* const order[] = {"VERY_HIGH_GPU_MEMORY", "HIGH_GPU_TEMPERATURE", "HIGH_GPU_MEMORY",
                                      "HIGH_GPU_POWER", "HIGH_HOST_MEMORY", "HIGH_CPU", "LOW_GPU_UTILIZATION"};
  for (int k = 0; k < 7; ++k)
    if (kind == order[k]) return k;
  return 999;
}

int sys_severity(const S& sev) { return sev == "crit" ? 2 : sev == "warn" ? 1 : 0; }  // common.py:98-102

}  // namespace

// diagnose_system over the engine's one node (diagnostics/system/api.py:189-209): the node's
// rules, scoped to the node; without an issue the cluster-level default primary.  Also emits
// SystemSummaryAgg and the PerGPUSummary rows (reporting/sections/system/model.py:50-117).
extern "C" int tml_diag_system(const tml_sys_diag_in* in, char* json_out, size_t cap) {
  tml_json::Scope json_scope;
  if (!in) return TML_ERR_ARG;
  std::vector<Issue> issues;
  sys_node_issues(in, issues);
  const S primary = sys_primary(issues, (long long)in->agg.n, in->agg);
  std::vector<S> is;
  for (const Issue& i : issues) is.push_back(i.json());
  return emit(Obj().kv("primary", primary).kv("issues", jarr(is)).kv("aggregate", sys_agg_json(in->agg))
                  .kv("per_gpu", sys_per_gpu_json(in->agg)).done(),
              json_out, cap);
}

// The same over several nodes (api.py:189-209): every node's issues, sorted by _issue_sort_key
// (priority, severity, score, node label as a string); a stable sort over the nodes in label
// order, as the reference sorts its list built in that order.
extern "C" int tml_diag_system_cluster(const tml_sys_diag_in* nodes, uint32_t n_nodes, const tml_sys_agg* cluster,
                                       char* json_out, size_t cap) {
  tml_json::Scope json_scope;
  if ((!nodes && n_nodes) || !cluster || n_nodes > TML_MAX_RANKS) return TML_ERR_ARG;
  struct Tagged { Issue issue; S label; long long samples; };
  std::vector<Tagged> all;
  Obj per_node;
  for (uint32_t k = 0; k < n_nodes; ++k) {
    const tml_sys_diag_in& in = nodes[k];
    char label_buf[33];
    memcpy(label_buf, in.node_label, 32);
    label_buf[32] = 0;
    std::vector<Issue> issues;
    sys_node_issues(&in, issues);
    for (Issue& i : issues) all.push_back({i, S(label_buf), (long long)in.agg.n});
    per_node.kv(label_buf, Obj().kv("aggregate", sys_agg_json(in.agg)).kv("per_gpu", sys_per_gpu_json(in.agg)).done());
  }
  std::stable_sort(all.begin(), all.end(), [](const Tagged& x, const Tagged& y) {
    const int px = sys_priority(x.issue.kind), py = sys_priority(y.issue.kind);
    if (px != py) return px < py;
    const int sx = sys_severity(x.issue.severity), sy = sys_severity(y.issue.severity);
    if (sx != sy) return sx > sy;
    if (x.issue.score != y.issue.score) return x.issue.score > y.issue.score;
    return strcmp(x.label.c_str(), y.label.c_str()) < 0;
  });
  std::vector<Issue> issues;
  for (const Tagged& t : all) issues.push_back(t.issue);
  const S primary = sys_primary(issues, all.empty() ? 0 : all[0].samples, *cluster);
  std::vector<S> is;
  for (const Issue& i : issues) is.push_back(i.json());
  return emit(Obj().kv("primary", primary).kv("issues", jarr(is)).kv("aggregate", sys_agg_json(*cluster))
                  .kv("nodes", per_node.done()).done(),
              json_out, cap);
}
