// Live "step combined" path: the render-tick twin of the window reduce.
// Included at the end of tml_engine.cu (one translation unit: it shares tml_ctx,
// ns_to_ms, the K3c scan kernels and the error plumbing).
//
// Replaces StepCombinedComputer._compute_impl of the reference
// (renderers/step_time/compute.py:129-315, 352-416, 452-470, 502-626): the last
// `lookback` records of the HBM ring -> 64-B rows, newest row of a step id wins,
// presence map -> cross-rank intersection -> last `window` common steps -> per-rank
// window SUMS of the six raw phases (ascending step order, like the reference's loop)
// and, after one row exchange, the per-step median / worst / sum series.
//
// The windows are a few hundred rows: these kernels are latency-, not bandwidth-bound;
// what matters is that the tick never touches the training stream and costs the host
// a handful of launches + two small synchronisations.  It may run on any stream,
// concurrently with the step path: the ring head is read on the DEVICE.

#define CB_THREADS 128

struct CombAcc {  // integer results of k_comb_rows
  u64 lo, hi, ncand, n, viol, latest, head, first_step, inrange;
};

// one consistent view of the ring head for the whole tick: the step path may commit
// while k_comb_rows is running, and its threads must agree on first_k / n
__global__ void k_comb_head(const DevState* __restrict__ st, CombAcc* acc) { acc->head = st->head; }

// K7a: last `lookback` ring records -> rows / step ids / candidate flags.
__global__ void __launch_bounds__(CB_THREADS) k_comb_rows(
    StepRing ring, u32 lookback, u32 kind, tml_window_row* __restrict__ rows, u64* __restrict__ steps,
    u8* __restrict__ cand, CombAcc* acc) {
  const u64 head = acc->head;
  const u32 ring_slots = ring.slots;
  u64 n = head < (u64)ring_slots ? head : (u64)ring_slots;
  if (n > lookback) n = lookback;
  const u64 first_k = head - n;
  u64 lo = ~0ull, hi = 0, latest = 0;
  u32 nc = 0, viol = 0;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const u64 slot = (first_k + i) % ring_slots;
    const RingHot* r = &ring.hot[slot];
    const u64 step = r->step;
    tml_window_row o;
    o.dataloader = ns_to_ms(r->dl);
    o.h2d = ns_to_ms(ring.cold[slot].h2d);
    o.forward = ns_to_ms(r->fwd);
    o.backward = ns_to_ms(r->bwd);
    o.optimizer = ns_to_ms(r->opt);
    o.step_wall = ns_to_ms(r->wall);
    o.peak_alloc = (double)r->peak_alloc;
    o.peak_resv = (double)r->peak_resv;
    rows[i] = o;
    steps[i] = step;
    // "ORDER BY step DESC, id DESC" + first-wins == the newest row of a step id; the memory
    // view only sees rows whose peaks are not NULL (common.py:143-150): newest such row
    bool last_of_step = true;
    if (i + 1 < n) {
      const u64 nx = (first_k + i + 1) % ring_slots;
      last_of_step = ring.hot[nx].step != step || (kind == TML_KIND_MEM && ring.mem[nx] == 0);
    }
    if (kind == TML_KIND_MEM && ring.mem[slot] == 0) last_of_step = false;
    if (i > 0 && ring.hot[(first_k + i - 1) % ring_slots].step > step) ++viol;
    if (i == 0) acc->first_step = step;
    cand[i] = last_of_step ? 1 : 0;
    if (last_of_step) { lo = step < lo ? step : lo; hi = step > hi ? step : hi; ++nc; }
    latest = step > latest ? step : latest;
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    u64 t;
    t = __shfl_xor_sync(0xffffffffu, lo, m); lo = t < lo ? t : lo;
    t = __shfl_xor_sync(0xffffffffu, hi, m); hi = t > hi ? t : hi;
    t = __shfl_xor_sync(0xffffffffu, latest, m); latest = t > latest ? t : latest;
  }
  nc = __reduce_add_sync(0xffffffffu, nc);
  viol = __reduce_add_sync(0xffffffffu, viol);
  if ((threadIdx.x & 31) == 0) {
    if (nc) { atomicMin(&acc->lo, lo); atomicMax(&acc->hi, hi); atomicAdd(&acc->ncand, (u64)nc); }
    if (viol) atomicAdd(&acc->viol, (u64)viol);
    atomicMax(&acc->latest, latest);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) acc->n = n;
}

// K7b: presence bytes of the candidates over [glo, glo + span).  Two launches: count the
// in-range candidates, then scatter -- or, for the memory view, write all ones when there
// are none: such a rank is absent from the reference's rank maps and must not constrain
// the intersection (common.py:143-178, 262-275).
__global__ void k_comb_inrange(const u64* __restrict__ steps, const u8* __restrict__ cand, CombAcc* acc,
                               u64 glo, u64 span) {
  const u64 n = acc->n;
  u32 c = 0;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
    if (cand[i]) { const u64 s = steps[i]; c += (s >= glo && (s - glo) < span) ? 1u : 0u; }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&acc->inrange, (u64)c);
}

__global__ void k_comb_presence(const u64* __restrict__ steps, const u8* __restrict__ cand,
                                const CombAcc* __restrict__ acc, u64 glo, u64 span, u32 ones_if_none,
                                u8* __restrict__ presence, u32* __restrict__ rowof) {
  const u64 n = acc->n;
  if (acc->inrange == 0 && ones_if_none) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < span; i += (u64)gridDim.x * blockDim.x)
      presence[i] = 1;
    return;
  }
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    if (cand[i]) {
      const u64 s = steps[i];
      if (s >= glo && (s - glo) < span) { presence[s - glo] = 1; rowof[s - glo] = (u32)i; }
    }
  }
}

// K7c: gather the selected rows (thread = 16-B chunk) ...
__global__ void k_comb_gather(const tml_window_row* __restrict__ rows, const u32* __restrict__ sel,
                              const u64* __restrict__ total_p, u64 window, const CombAcc* __restrict__ acc,
                              tml_window_row* __restrict__ xrows) {
  if (acc->inrange == 0) return;
  const u64 total = *total_p;
  const u64 keep = total < window ? total : window;
  const uint4* src = reinterpret_cast<const uint4*>(rows);
  uint4* dst = reinterpret_cast<uint4*>(xrows);
  for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < keep * 4; t += (u64)gridDim.x * blockDim.x)
    dst[t] = src[(u64)sel[t >> 2] * 4 + (t & 3)];
}

// ... and sum the six raw phases in ascending step order, one lane per phase: the
// reference adds `for step in steps` (compute.py:517-524), and the rank tie-breaks
// downstream (argmax, closest-to-median) are decided by the last ulp of these sums.
// Lanes 6, 7: the rank's peak over the window (max of peak_alloc / peak_resv, common.py:289).
__global__ void __launch_bounds__(32) k_comb_sums(const tml_window_row* __restrict__ xrows,
                                                  const u64* __restrict__ total_p, u64 window,
                                                  const CombAcc* __restrict__ cacc,
                                                  double* __restrict__ out) {
  const u64 total = *total_p;
  const u64 keep = total < window ? total : window;
  const int lane = threadIdx.x;
  if (lane >= 8) return;
  if (lane == 0) out[8] = (double)cacc->inrange;
  if (cacc->inrange == 0) { out[lane] = 0.0; return; }
  const double* p = reinterpret_cast<const double*>(xrows) + lane;
  double acc = lane < 6 ? 0.0 : -INFINITY;
  // the loads are independent of the chain: unrolled so eight are in flight per DADD run
  if (lane < 6) {
#pragma unroll 8
    for (u64 j = 0; j < keep; ++j) acc += __ldg(&p[j * 8]);
  } else {
#pragma unroll 8
    for (u64 j = 0; j < keep; ++j) acc = fmax(acc, __ldg(&p[j * 8]));
  }
  out[lane] = acc;
}

struct CombSeriesParams {
  const double* rows[TML_MAX_RANKS];
  double* series;  // [n_cols][3: median, worst, sum][n]
  u64 n;
  u32 n_ranks;
  u32 first_col, n_cols;
};

// K7d: per-step median / worst / sum across ranks for the six raw phases
// (compute.py:573-596).  thread = (step, phase); sum runs in rank order like np.sum
// over a < 8-element array... and pairwise above: see comb_sum.
__device__ __forceinline__ double comb_sum(const double* v, int n) {
  // numpy's pairwise_sum for a contiguous f64 array: plain loop below 8 elements,
  // 8 running partials (combined as ((r0+r1)+(r2+r3)) + ((r4+r5)+(r6+r7))) up to the
  // 128-element block; TML_MAX_RANKS = 64 never reaches the recursive split.
  if (n < 8) {
    double s = 0.0;  // numpy starts from 0.0 (its -0.0 start only matters for empty sums)
    for (int i = 0; i < n; ++i) s += v[i];
    return s;
  }
  double r[8];
  for (int k = 0; k < 8; ++k) r[k] = v[k];
  int i = 8;
  for (; i + 8 <= n; i += 8)
    for (int k = 0; k < 8; ++k) r[k] += v[i + k];
  double s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) s += v[i];
  return s;
}

__global__ void __launch_bounds__(CB_THREADS) k_comb_series(const __grid_constant__ CombSeriesParams p) {
  const int R = (int)p.n_ranks;
  const u64 nc = p.n_cols;
  const u64 work = p.n * nc;
  for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < work; t += (u64)gridDim.x * blockDim.x) {
    const u64 j = t / nc;
    const int m = (int)(t - j * nc);
    double v[TML_MAX_RANKS];
    for (int r = 0; r < R; ++r) v[r] = p.rows[r][j * 8 + p.first_col + m];
    const double sum = comb_sum(v, R);
    for (int a = 1; a < R; ++a) {  // insertion sort (R <= 64, usually <= 8)
      const double key = v[a];
      int b = a - 1;
      while (b >= 0 && v[b] > key) { v[b + 1] = v[b]; --b; }
      v[b + 1] = key;
    }
    const double med = (R & 1) ? v[R / 2] : (v[R / 2 - 1] + v[R / 2]) * 0.5;
    double* S = p.series + (u64)m * 3ull * p.n;
    S[j] = med;
    S[p.n + j] = v[R - 1];
    S[2 * p.n + j] = sum;
  }
}

struct CombWs {
  u64 cap = 0, cap_span = 0;
  tml_window_row* d_rows = nullptr;
  tml_window_row* d_x = nullptr;
  u64* d_steps = nullptr;
  u8* d_cand = nullptr;
  u32* d_rowof = nullptr;
  u32* d_selrow = nullptr;
  u64* d_selstep = nullptr;
  u32* d_blockcnt = nullptr;
  u64 cap_blk = 0;
  u64* d_total = nullptr;
  CombAcc* d_acc = nullptr;
  double* d_sums = nullptr;
  void* h_stage = nullptr;  // pinned, private: a tick may overlap a final-summary reduce
  u64 n = 0, ncand = 0, n_common = 0, n_rows = 0;
  u32 kind = 0;
  bool ready = false;
};

static int comb_ws(tml_ctx* c, u32 kind, CombWs** out) {
  if (!c->comb[kind]) {
    CombWs* w = new CombWs();
    CK(cudaMalloc(&w->d_total, sizeof(u64)));
    CK(cudaMalloc(&w->d_acc, sizeof(CombAcc)));
    CK(cudaMalloc(&w->d_sums, 16 * sizeof(double)));
    CK(cudaHostAlloc(&w->h_stage, 1024, cudaHostAllocDefault));
    c->comb[kind] = w;
  }
  *out = (CombWs*)c->comb[kind];
  return TML_OK;
}

static void comb_free_one(tml_ctx* c, u32 kind) {
  CombWs* w = (CombWs*)c->comb[kind];
  if (!w) return;
  cudaFree(w->d_rows); cudaFree(w->d_x); cudaFree(w->d_steps); cudaFree(w->d_cand);
  cudaFree(w->d_rowof); cudaFree(w->d_selrow); cudaFree(w->d_selstep); cudaFree(w->d_blockcnt);
  cudaFree(w->d_total); cudaFree(w->d_acc); cudaFree(w->d_sums);
  cudaFreeHost(w->h_stage);
  delete w;
  c->comb[kind] = nullptr;
}

static void comb_free(tml_ctx* c) { comb_free_one(c, 0); comb_free_one(c, 1); }

extern "C" {

int tml_combined_prepare(tml_ctx* c, uint32_t kind, uint32_t lookback, void* stream,
                         tml_combined_info* out) {
  if (!c || !out || lookback == 0 || kind > 1) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  memset(out, 0, sizeof(*out));
  CombWs* w = nullptr;
  int rc = comb_ws(c, kind, &w);
  if (rc != TML_OK) return rc;
  // keep clear of the slots the step path may be rewriting while the tick runs
  u64 lb = lookback;
  const u64 safe = c->ring_slots > TML_N_EPOCHS ? c->ring_slots - TML_N_EPOCHS : 1;
  if (lb > safe) lb = safe;
  if (lb > w->cap) {
    cudaFree(w->d_rows); cudaFree(w->d_x); cudaFree(w->d_steps); cudaFree(w->d_cand);
    cudaFree(w->d_selrow); cudaFree(w->d_selstep);
    w->d_rows = w->d_x = nullptr; w->d_steps = w->d_selstep = nullptr; w->d_cand = nullptr;
    w->d_selrow = nullptr; w->cap = 0;
    CK(cudaMalloc(&w->d_rows, (size_t)lb * sizeof(tml_window_row)));
    CK(cudaMalloc(&w->d_x, (size_t)lb * sizeof(tml_window_row)));
    CK(cudaMalloc(&w->d_steps, (size_t)lb * sizeof(u64)));
    CK(cudaMalloc(&w->d_cand, (size_t)lb));
    CK(cudaMalloc(&w->d_selrow, (size_t)lb * sizeof(u32)));
    CK(cudaMalloc(&w->d_selstep, (size_t)lb * sizeof(u64)));
    w->cap = lb;
  }
  CombAcc init;
  memset(&init, 0, sizeof(init));
  init.lo = ~0ull;
  CK(cudaMemcpyAsync(w->d_acc, &init, sizeof(init), cudaMemcpyHostToDevice, s));
  int grid = (int)((lb + CB_THREADS - 1) / CB_THREADS);
  if (grid > c->n_sms) grid = c->n_sms;
  k_comb_head<<<1, 1, 0, s>>>(c->d_state, w->d_acc);
  CK(cudaPeekAtLastError());
  k_comb_rows<<<grid, CB_THREADS, 0, s>>>(c->ring, (u32)lb, kind, w->d_rows, w->d_steps,
                                          w->d_cand, w->d_acc);
  CK(cudaPeekAtLastError());
  c->launches += 2;
  CK(cudaMemcpyAsync(w->h_stage, w->d_acc, sizeof(CombAcc), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CombAcc acc;
  memcpy(&acc, w->h_stage, sizeof(acc));
  w->n = acc.n; w->ncand = acc.ncand; w->n_common = 0; w->ready = true; w->kind = kind;
  out->n_rows = acc.n;
  out->n_cand = acc.ncand;
  out->lo = acc.ncand ? acc.lo : 0;
  out->hi = acc.ncand ? acc.hi : 0;
  out->latest_step = acc.latest;
  out->first_step = acc.n ? acc.first_step : 0;
  out->truncated = acc.head > acc.n ? 1u : 0u;
  out->monotone = acc.viol == 0 ? 1u : 0u;
  if (acc.viol)
    return set_err(TML_ERR_NONMONOTONIC, "step ids decrease inside the look-back rows (%llu places)",
                   (unsigned long long)acc.viol);
  return TML_OK;
}

int tml_combined_presence(tml_ctx* c, uint32_t kind, uint64_t glo, uint64_t span, uint8_t* presence,
                          void* stream) {
  if (!c || !presence || span == 0 || kind > 1) return TML_ERR_ARG;
  CombWs* w = (CombWs*)c->comb[kind];
  if (!w || !w->ready) return set_err(TML_ERR_STATE, "tml_combined_presence before tml_combined_prepare");
  if (span >> 32) return set_err(TML_ERR_UNSUPPORTED, "step-id span %llu too wide", (u64)span);
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  int rc = ensure(&w->d_rowof, &w->cap_span, span);
  if (rc != TML_OK) return rc;
  if (w->n == 0) { CK(cudaMemsetAsync(presence, 1, span, s)); return TML_OK; }  // no rows: not a rank yet
  CK(cudaMemsetAsync(presence, 0, span, s));
  CK(cudaMemsetAsync(&w->d_acc->inrange, 0, sizeof(u64), s));
  int grid = (int)((w->n + 255) / 256);
  if (grid > c->n_sms) grid = c->n_sms;
  k_comb_inrange<<<grid, 256, 0, s>>>(w->d_steps, w->d_cand, w->d_acc, glo, span);
  CK(cudaPeekAtLastError());
  int pgrid = (int)(((w->n > span ? w->n : span) + 255) / 256);
  if (pgrid > c->n_sms) pgrid = c->n_sms;
  k_comb_presence<<<pgrid, 256, 0, s>>>(w->d_steps, w->d_cand, w->d_acc, glo, span,
                                        kind == TML_KIND_MEM ? 1u : 0u, presence, w->d_rowof);
  CK(cudaPeekAtLastError());
  c->launches += 2;
  return TML_OK;
}

int tml_combined_select(tml_ctx* c, uint32_t kind, uint64_t glo, uint64_t span, const uint8_t* presence,
                        uint32_t window, void* stream, tml_combined_align* out) {
  if (!c || !out || window == 0 || kind > 1) return TML_ERR_ARG;
  CombWs* w = (CombWs*)c->comb[kind];
  if (!w || !w->ready) return set_err(TML_ERR_STATE, "tml_combined_select before tml_combined_prepare");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  memset(out, 0, sizeof(*out));
  w->n_common = 0; w->n_rows = 0;
  if (span == 0 || !presence) return TML_OK;
  const u32 nb = (u32)((span + SEL_TILE - 1) / SEL_TILE);
  int rc = ensure(&w->d_blockcnt, &w->cap_blk, nb);
  if (rc != TML_OK) return rc;
  k_sel_count<<<nb, SEL_THREADS, 0, s>>>(presence, span, w->d_blockcnt);
  CK(cudaPeekAtLastError());
  k_sel_scan<<<1, 1024, 0, s>>>(w->d_blockcnt, nb, w->d_total);
  CK(cudaPeekAtLastError());
  c->launches += 2;
  char* st = (char*)w->h_stage;
  if (w->n == 0) {  // this rank owns no rows: only the count is needed (identical everywhere)
    CK(cudaMemcpyAsync(st, w->d_total, sizeof(u64), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    u64 total = 0;
    memcpy(&total, st, sizeof(u64));
    out->n_common = total < window ? total : window;
    w->n_common = out->n_common;
    return TML_OK;
  }
  // a rank without in-range candidates wrote all ones: its rowof is stale, and the gather /
  // sums kernels skip themselves on acc->inrange == 0.  The intersection never holds more
  // steps than an owning rank has candidates (<= cap).
  k_sel_scatter<<<nb, SEL_THREADS, 0, s>>>(presence, span, w->d_blockcnt, w->d_total,
                                           (u64)(window < w->cap ? window : w->cap), glo,
                                           w->d_rowof, w->d_selrow, w->d_selstep);
  CK(cudaPeekAtLastError());
  const u64 maxkeep = w->ncand < window ? w->ncand : window;
  int grid = (int)((maxkeep * 4 + 255) / 256);
  if (grid < 1) grid = 1;
  if (grid > c->n_sms) grid = c->n_sms;
  k_comb_gather<<<grid, 256, 0, s>>>(w->d_rows, w->d_selrow, w->d_total, (u64)window, w->d_acc, w->d_x);
  CK(cudaPeekAtLastError());
  k_comb_sums<<<1, 32, 0, s>>>(w->d_x, w->d_total, (u64)window, w->d_acc, w->d_sums);
  CK(cudaPeekAtLastError());
  c->launches += 3;
  CK(cudaMemcpyAsync(st, w->d_total, sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(st + 64, w->d_sums, 9 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  u64 total = 0;
  memcpy(&total, st, sizeof(u64));
  double f[9];
  memcpy(f, st + 64, sizeof(f));
  const u64 keep = total < window ? total : window;
  out->n_common = keep;
  w->n_common = keep;
  if (keep == 0 || f[8] == 0.0) return TML_OK;  // no in-range candidates: the rank owns no rows
  memcpy(out->sums, f, 6 * sizeof(double));
  out->peaks[0] = f[6]; out->peaks[1] = f[7];
  out->n_rows = keep;
  w->n_rows = keep;
  return TML_OK;
}

const void* tml_combined_rows(tml_ctx* c, uint32_t kind) {
  if (!c || kind > 1 || !c->comb[kind]) return nullptr;
  CombWs* w = (CombWs*)c->comb[kind];
  return w->n_rows ? w->d_x : nullptr;
}

int tml_combined_steps(tml_ctx* c, uint32_t kind, uint64_t* steps_host, uint64_t cap, void* stream) {
  if (!c || !steps_host || kind > 1) return TML_ERR_ARG;
  CombWs* w = (CombWs*)c->comb[kind];
  if (!w || !w->ready) return set_err(TML_ERR_STATE, "tml_combined_steps before tml_combined_select");
  if (w->n_rows == 0) return set_err(TML_ERR_STATE, "this rank holds no rows of the window");
  if (cap < w->n_common) return TML_ERR_SMALL;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(steps_host, w->d_selstep, (size_t)w->n_common * sizeof(u64), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return TML_OK;
}

int tml_combined_series(tml_ctx* c, const void* const* rank_rows, uint32_t n_ranks, uint64_t n_common,
                        uint32_t first_col, uint32_t n_cols, double* series_dev, void* stream) {
  if (!c || !rank_rows || !series_dev || n_ranks == 0 || n_ranks > TML_MAX_RANKS) return TML_ERR_ARG;
  if (n_cols == 0 || first_col + n_cols > 8) return TML_ERR_ARG;
  if (n_common == 0) return TML_OK;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(c->device));
  CombSeriesParams p;
  memset(&p, 0, sizeof(p));
  for (u32 r = 0; r < n_ranks; ++r) {
    if (!rank_rows[r]) return TML_ERR_ARG;
    p.rows[r] = (const double*)rank_rows[r];
  }
  p.series = series_dev;
  p.n = n_common;
  p.n_ranks = n_ranks;
  p.first_col = first_col;
  p.n_cols = n_cols;
  int grid = (int)((n_common * n_cols + CB_THREADS - 1) / CB_THREADS);
  if (grid > c->n_sms * 4) grid = c->n_sms * 4;
  k_comb_series<<<grid, CB_THREADS, 0, s>>>(p);
  CK(cudaPeekAtLastError());
  c->launches += 1;
  return TML_OK;
}

}  // extern "C"

// ============================================================================ layer time tick
// The live layer-time panel's device stages (include/traceml_b200.h, LAYER TIME TICK).  The layer
// ring is [ring_steps][n_layers] 48-B records; the snapshot gives a warp 32 consecutive layers
// (lane = layer) and walks the retained steps, so each step it loads is one contiguous 1.5-KB run.
// Like K7 these kernels run on the tick's own stream while the step path may commit: the head is
// read once on the device (k_lt_head) and the bounds and the snapshot both use that view.

#define LT_THREADS 128

struct LTickHdr {
  u64 head, n;                          // completed commits, retained steps (<= ring_steps)
  u64 fwd_rows, bwd_rows;               // 1 + newest position holding a forward / backward row; 0: none
  u64 newest_fwd, newest_bwd, oldest;   // step ids of those rows and of the oldest retained step
};

__global__ void k_lt_head(const u64* head, u32 ring_steps, LTickHdr* h) {
  const u64 v = *reinterpret_cast<const volatile u64*>(head);
  h->head = v;
  h->n = v < (u64)ring_steps ? v : (u64)ring_steps;
  h->fwd_rows = h->bwd_rows = 0;
}

// one warp per retained step: its step id and whether any layer has a forward / backward call
// (whether the reference's forward / backward table holds a row for it)
__global__ void __launch_bounds__(LT_THREADS) k_lt_rows(const tml_layer_record* __restrict__ ring, u32 n_layers,
                                                        u32 ring_steps, LTickHdr* h, u64* __restrict__ steps,
                                                        u8* __restrict__ dirs) {
  const u64 n = h->n, first = h->head - n;
  const u32 lane = threadIdx.x & 31;
  const u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
  for (u64 i = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
    const tml_layer_record* row = ring + ((first + i) % ring_steps) * (u64)n_layers;
    u64 calls = 0;  // fwd_calls | bwd_calls << 32
    for (u32 l = lane; l < n_layers; l += 32) calls |= *reinterpret_cast<const u64*>(&row[l].fwd_calls);
    const bool f = __any_sync(0xffffffffu, (u32)calls != 0u);
    const bool b = __any_sync(0xffffffffu, (u32)(calls >> 32) != 0u);
    if (lane == 0) {
      steps[i] = row[0].step;
      dirs[i] = (f ? 1 : 0) | (b ? 2 : 0);
      if (f) atomicMax(&h->fwd_rows, i + 1);
      if (b) atomicMax(&h->bwd_rows, i + 1);
    }
  }
}

__global__ void k_lt_bounds(LTickHdr* h, const u64* __restrict__ steps) {
  h->oldest = h->n ? steps[0] : 0;
  h->newest_fwd = h->fwd_rows ? steps[h->fwd_rows - 1] : 0;
  h->newest_bwd = h->bwd_rows ? steps[h->bwd_rows - 1] : 0;
}

__global__ void __launch_bounds__(LT_THREADS) k_lt_snap(const tml_layer_record* __restrict__ ring, u32 n_layers,
                                                        u32 ring_steps, const LTickHdr* __restrict__ h,
                                                        const u64* __restrict__ steps, const u8* __restrict__ dirs,
                                                        u64 safe, tml_layer_snap* __restrict__ out) {
  const u32 lane = threadIdx.x & 31;
  const u32 warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp * 32u >= n_layers) return;  // warp-uniform
  const u64 n = h->n, first = h->head - n;
  // per direction, over that direction's rows: lo = 1 + the newest with a step id < safe (where the
  // reference's backward scan stops), cur = the newest with step id == safe
  int lo0 = 0, lo1 = 0, cur0 = -1, cur1 = -1;
  for (u32 i = lane; i < (u32)n; i += 32) {
    const u64 s = steps[i];
    const u32 d = dirs[i];
    if (d & 1u) { if (s < safe) lo0 = (int)i + 1; else if (s == safe) cur0 = (int)i; }
    if (d & 2u) { if (s < safe) lo1 = (int)i + 1; else if (s == safe) cur1 = (int)i; }
  }
  lo0 = __reduce_max_sync(0xffffffffu, lo0); lo1 = __reduce_max_sync(0xffffffffu, lo1);
  cur0 = __reduce_max_sync(0xffffffffu, cur0); cur1 = __reduce_max_sync(0xffffffffu, cur1);
  const bool has0 = cur0 >= lo0, has1 = cur1 >= lo1;  // else the rank is missing in that direction
  const u32 l = warp * 32u + lane;
  if (l >= n_layers) return;
  u64 cf = 0, cb = 0, pf = 0, pb = 0;
  u32 flags = (has0 ? TML_LSNAP_RANK_FWD : 0u) | (has1 ? TML_LSNAP_RANK_BWD : 0u), lf = 0, lb = 0;
  if (has0 || has1) {
    const u32 start = (u32)(has0 && has1 ? min(lo0, lo1) : has0 ? lo0 : lo1);
#pragma unroll 4
    for (u32 i = start; i < (u32)n; ++i) {
      const tml_layer_record* r = ring + ((first + i) % ring_steps) * (u64)n_layers + l;
      const u64 fns = r->fwd_ns, bns = r->bwd_ns;
      const u64 calls = *reinterpret_cast<const u64*>(&r->fwd_calls);
      if (has0 && (int)i >= lo0 && (u32)calls != 0u) {
        pf = fns > pf ? fns : pf;
        lf = i;
        flags |= TML_LSNAP_PEAK_FWD;
        if ((int)i == cur0) { cf = fns; flags |= TML_LSNAP_CUR_FWD; }
      }
      if (has1 && (int)i >= lo1 && (u32)(calls >> 32) != 0u) {
        pb = bns > pb ? bns : pb;
        lb = i;
        flags |= TML_LSNAP_PEAK_BWD;
        if ((int)i == cur1) { cb = bns; flags |= TML_LSNAP_CUR_BWD; }
      }
    }
  }
  tml_layer_snap o;
  o.cur_fwd_ns = cf; o.cur_bwd_ns = cb; o.peak_fwd_ns = pf; o.peak_bwd_ns = pb;
  o.flags = flags; o.last_fwd = lf; o.last_bwd = lb; o._pad = 0;
  out[l] = o;
}

// wire_rows' float(int(ns)) / 1.0e6, the point where the reference's values become floats:
// ns_to_ms is that correctly rounded quotient without the division's slow-path call
__device__ __forceinline__ double lt_ms(u64 ns) { return ns_to_ms(ns); }

// one direction of one layer on one rank: max over ranks (from 0.0, like the reference's
// dict.get(k, 0.0)) and the first rank that has a current / a peak value
struct LtDir {
  double cur = 0.0, peak = 0.0;
  u32 cur_rank = 0, peak_rank = 0, peak_last = 0;
  bool has_cur = false, has_peak = false;
  __device__ __forceinline__ void add(u32 r, bool c, u64 cur_ns, bool p, u64 peak_ns, u32 last) {
    if (c) {
      const double v = lt_ms(cur_ns);
      cur = v > cur ? v : cur;
      if (!has_cur) cur_rank = r;
      has_cur = true;
    }
    if (p) {
      const double v = lt_ms(peak_ns);
      peak = v > peak ? v : peak;
      if (!has_peak) { peak_rank = r; peak_last = last; }
      has_peak = true;
    }
  }
};

// one thread per layer over the R gathered snapshots (rank order)
__global__ void __launch_bounds__(LT_THREADS) k_lt_fold(const tml_layer_snap* __restrict__ snaps, u32 n_ranks,
                                                        u32 n_layers, tml_layer_tick_row* __restrict__ out,
                                                        u32* __restrict__ rank_flags) {
  if (blockIdx.x == 0)
    for (u32 r = threadIdx.x; r < n_ranks; r += blockDim.x)
      rank_flags[r] = snaps[(u64)r * n_layers].flags & (TML_LSNAP_RANK_FWD | TML_LSNAP_RANK_BWD);
  const u32 l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n_layers) return;
  LtDir f, b;
  // worst rank (compute.py:239-253): `totals` gets the ranks with a current forward value in rank
  // order, then the ranks with only a backward one; a rank's total is fwd + bwd in that order, and
  // max(totals.items(), key=...) keeps the FIRST maximum -- so only a strictly larger total wins
  int worst = -1;
  double wv = 0.0;
  for (u32 r = 0; r < n_ranks; ++r) {
    const tml_layer_snap* s = &snaps[(u64)r * n_layers + l];
    const u32 fl = s->flags;
    const u64 cfn = s->cur_fwd_ns, cbn = s->cur_bwd_ns;
    f.add(r, fl & TML_LSNAP_CUR_FWD, cfn, fl & TML_LSNAP_PEAK_FWD, s->peak_fwd_ns, s->last_fwd);
    b.add(r, fl & TML_LSNAP_CUR_BWD, cbn, fl & TML_LSNAP_PEAK_BWD, s->peak_bwd_ns, s->last_bwd);
    if (fl & TML_LSNAP_CUR_FWD) {
      double t = lt_ms(cfn);
      if (fl & TML_LSNAP_CUR_BWD) t = t + lt_ms(cbn);
      if (worst < 0 || t > wv) { worst = (int)r; wv = t; }
    }
  }
  for (u32 r = 0; r < n_ranks; ++r) {
    const tml_layer_snap* s = &snaps[(u64)r * n_layers + l];
    if ((s->flags & (TML_LSNAP_CUR_FWD | TML_LSNAP_CUR_BWD)) == TML_LSNAP_CUR_BWD) {
      const double t = lt_ms(s->cur_bwd_ns);
      if (worst < 0 || t > wv) { worst = (int)r; wv = t; }
    }
  }
  tml_layer_tick_row o;
  o.cur_fwd_ms = f.cur; o.cur_bwd_ms = b.cur; o.peak_fwd_ms = f.peak; o.peak_bwd_ms = b.peak;
  o.worst_rank = worst;
  o.flags = (f.has_cur ? TML_LSNAP_CUR_FWD : 0u) | (b.has_cur ? TML_LSNAP_CUR_BWD : 0u)
          | (f.has_peak ? TML_LSNAP_PEAK_FWD : 0u) | (b.has_peak ? TML_LSNAP_PEAK_BWD : 0u);
  o.peak_last[0] = f.peak_last; o.peak_last[1] = b.peak_last;
  o.cur_rank[0] = (uint16_t)f.cur_rank; o.cur_rank[1] = (uint16_t)b.cur_rank;
  o.peak_rank[0] = (uint16_t)f.peak_rank; o.peak_rank[1] = (uint16_t)b.peak_rank;
  out[l] = o;
}

struct LTickWs {
  u64 cap = 0;
  u64* d_steps = nullptr;
  u8* d_dirs = nullptr;
  LTickHdr* d_hdr = nullptr;
  LTickHdr* h_hdr = nullptr;  // pinned
  u32 n_layers = 0, ring_steps = 0;  // the layer ring the bounds were taken on
  bool ready = false;
};

static void ltick_free(tml_ctx* c) {
  LTickWs* w = (LTickWs*)c->ltick;
  if (!w) return;
  cudaFree(w->d_steps); cudaFree(w->d_dirs); cudaFree(w->d_hdr);
  cudaFreeHost(w->h_hdr);
  delete w;
  c->ltick = nullptr;
}

extern "C" {

int tml_layer_tick_bounds(tml_ctx* c, uint64_t* newest_fwd_step, uint64_t* newest_bwd_step,
                          uint64_t* oldest_step, void* stream) {
  if (!c || !newest_fwd_step || !newest_bwd_step || !oldest_step) return TML_ERR_ARG;
  if (!c->n_layers) return set_err(TML_ERR_STATE, "tml_layer_tick_bounds before tml_layer_init");
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  if (!c->ltick) {
    LTickWs* w = new LTickWs();
    c->ltick = w;
    CK(cudaMalloc(&w->d_hdr, sizeof(LTickHdr)));
    CK(cudaHostAlloc(&w->h_hdr, sizeof(LTickHdr), cudaHostAllocDefault));
  }
  LTickWs* w = (LTickWs*)c->ltick;
  w->ready = false;
  if (w->cap < c->layer_steps) {
    cudaFree(w->d_steps); cudaFree(w->d_dirs);
    w->d_steps = nullptr; w->d_dirs = nullptr; w->cap = 0;
    CK(cudaMalloc(&w->d_steps, (size_t)c->layer_steps * sizeof(u64)));
    CK(cudaMalloc(&w->d_dirs, (size_t)c->layer_steps));
    w->cap = c->layer_steps;
  }
  k_lt_head<<<1, 1, 0, s>>>(c->d_layer_head, c->layer_steps, w->d_hdr);
  CK(cudaPeekAtLastError());
  int grid = (int)(((u64)c->layer_steps * 32 + LT_THREADS - 1) / LT_THREADS);
  if (grid > c->n_sms * 4) grid = c->n_sms * 4;
  k_lt_rows<<<grid, LT_THREADS, 0, s>>>(c->d_layer_ring, c->n_layers, c->layer_steps, w->d_hdr, w->d_steps,
                                        w->d_dirs);
  CK(cudaPeekAtLastError());
  k_lt_bounds<<<1, 1, 0, s>>>(w->d_hdr, w->d_steps);
  CK(cudaPeekAtLastError());
  c->launches += 3;
  CK(cudaMemcpyAsync(w->h_hdr, w->d_hdr, sizeof(LTickHdr), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  const LTickHdr h = *w->h_hdr;
  *newest_fwd_step = h.newest_fwd;
  *newest_bwd_step = h.newest_bwd;
  *oldest_step = h.oldest;
  w->n_layers = c->n_layers; w->ring_steps = c->layer_steps; w->ready = true;
  return (h.fwd_rows ? TML_LAYER_HAS_FWD : 0) | (h.bwd_rows ? TML_LAYER_HAS_BWD : 0);
}

int tml_layer_tick_snapshot(tml_ctx* c, uint64_t safe_step, void* out_dev, void* stream) {
  if (!c || !out_dev) return TML_ERR_ARG;
  LTickWs* w = (LTickWs*)c->ltick;
  if (!w || !w->ready || w->n_layers != c->n_layers || w->ring_steps != c->layer_steps)
    return set_err(TML_ERR_STATE, "tml_layer_tick_snapshot without tml_layer_tick_bounds on this layer ring");
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  const u64 warps = ((u64)c->n_layers + 31) / 32;
  const int grid = (int)((warps * 32 + LT_THREADS - 1) / LT_THREADS);
  k_lt_snap<<<grid, LT_THREADS, 0, s>>>(c->d_layer_ring, c->n_layers, c->layer_steps, w->d_hdr, w->d_steps,
                                        w->d_dirs, safe_step, (tml_layer_snap*)out_dev);
  CK(cudaPeekAtLastError());
  c->launches += 1;
  return TML_OK;
}

int tml_layer_tick_fold(tml_ctx* c, const void* snaps_dev, uint32_t n_ranks, uint32_t n_layers, void* out_dev,
                        void* stream) {
  if (!c || !snaps_dev || !out_dev || n_ranks == 0 || n_ranks > 0xffffu || n_layers == 0) return TML_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  tml_layer_tick_row* rows = (tml_layer_tick_row*)out_dev;
  const int grid = (int)(((u64)n_layers + LT_THREADS - 1) / LT_THREADS);
  k_lt_fold<<<grid, LT_THREADS, 0, s>>>((const tml_layer_snap*)snaps_dev, n_ranks, n_layers, rows,
                                        reinterpret_cast<u32*>(rows + n_layers));
  CK(cudaPeekAtLastError());
  c->launches += 1;
  return TML_OK;
}

int tml_layer_load_(tml_ctx* c, const tml_layer_record* recs, uint64_t n_steps, void* stream) {
  if (!c || (!recs && n_steps)) return TML_ERR_ARG;
  if (!c->n_layers) return set_err(TML_ERR_STATE, "tml_layer_load_ before tml_layer_init");
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard dg(c);
  const u64 L = c->n_layers, keep = n_steps < (u64)c->layer_steps ? n_steps : (u64)c->layer_steps;
  for (u64 k = n_steps - keep; k < n_steps; ++k)
    CK(cudaMemcpyAsync(c->d_layer_ring + (k % c->layer_steps) * L, recs + k * L, L * sizeof(tml_layer_record),
                       cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(c->d_layer_head, &n_steps, sizeof(u64), cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s));
  c->layer_commits = n_steps;
  c->layer_tail = 0;
  return TML_OK;
}

}  // extern "C"
