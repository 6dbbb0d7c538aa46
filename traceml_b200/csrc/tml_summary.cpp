// tml_reduce_run: the cross-rank window reduce sequenced natively (one rank per process).
//
// Written against the library's own public stages (include/traceml_b200.h) plus NCCL on
// the communicator the host hands in.  It mirrors traceml_b200/reduce.py stage for
// stage -- that module stays as the multi-engine (several ranks in one process) driver
// the single-GPU parity tests use, and as the executable specification of this file.
//
// Why native: at R >= 2 the reduce is latency-bound (three small exchanges + five
// kernel launches around two short bandwidth kernels); the interpreter between the
// stages cost more than the kernels.  Here an exchange is
// pinned-buffer H2D + ncclAllGather + D2H + one stream sync.
//
// NCCL is resolved at run time from the copy the process already has loaded (the one
// torch.distributed uses): no link-time dependency, no second NCCL in the process.

#include <dlfcn.h>
#include <fcntl.h>
#include <nccl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>

#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/traceml_b200.h"
#include "tml_internal.h"

namespace {

typedef uint64_t u64;
typedef uint32_t u32;

// ------------------------------------------------------------------ NCCL, late-bound
struct Nccl {
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t,
                            cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};

Nccl g_nccl;
std::once_flag g_nccl_once;

void load_nccl() {
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // torch's copy, already mapped
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return;
#define TML_SYM(field, name) *(void**)(&g_nccl.field) = dlsym(h, name)
  TML_SYM(AllGather, "ncclAllGather");
  TML_SYM(AllReduce, "ncclAllReduce");
  TML_SYM(Send, "ncclSend");
  TML_SYM(Recv, "ncclRecv");
  TML_SYM(GroupStart, "ncclGroupStart");
  TML_SYM(GroupEnd, "ncclGroupEnd");
  TML_SYM(GetErrorString, "ncclGetErrorString");
#undef TML_SYM
  g_nccl.ok = g_nccl.AllGather && g_nccl.AllReduce && g_nccl.Send && g_nccl.Recv && g_nccl.GroupStart &&
              g_nccl.GroupEnd && g_nccl.GetErrorString;
}

#define CKC(call)                                                                                \
  do {                                                                                           \
    cudaError_t e_ = (call);                                                                     \
    if (e_ != cudaSuccess)                                                                       \
      return tml_set_error_(TML_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                            __FILE__, __LINE__);                                                 \
  } while (0)
#define CKN(call)                                                                                  \
  do {                                                                                             \
    ncclResult_t r_ = (call);                                                                      \
    if (r_ != ncclSuccess)                                                                         \
      return tml_set_error_(TML_ERR_CUDA, "%s failed: %s (%s:%d)", #call, g_nccl.GetErrorString(r_), \
                            __FILE__, __LINE__);                                                   \
  } while (0)
#define CKT(call)                 \
  do {                            \
    int rc_ = (call);             \
    if (rc_ != TML_OK) return rc_; \
  } while (0)

// ------------------------------------------------------------------ per-context workspace
constexpr int XV = 160;  // doubles per rank in a small exchange (largest: 23 + 17 + 24 = 64; bands 128)

struct RunWs {
  double* d_send = nullptr;  // XV doubles
  double* d_recv = nullptr;  // TML_MAX_RANKS * XV
  double* h_send = nullptr;  // pinned
  double* h_recv = nullptr;
  uint8_t* d_presence = nullptr;
  u64 cap_presence = 0;
  double* d_series[2] = {nullptr, nullptr};
  u64 cap_series[2] = {0, 0};
  char* d_recv_rows = nullptr;  // a2a: my shard of every rank's rows
  u64 cap_recv_rows = 0;
  char* d_zero_rows = nullptr;  // a2a: what a rank outside `used` sends
  u64 cap_zero_rows = 0;
  bool p2p_warm = false;  // peer mappings already open: peer loads cost nothing extra
  cudaStream_t side = nullptr;  // process aggregates (K6) run beside K3a, not in front of it
  cudaEvent_t side_gate = nullptr;  // side waits for what `stream` held at entry (ring loads)
  // host mailbox for the small exchanges (ranks of one node): see Run::xchg
  bool mbox_tried = false;
  void* mbox = nullptr;
  size_t mbox_bytes = 0;
  u64 mbox_seq = 0;
};

// ------------------------------------------------------------------ host mailbox
// The small exchanges carry HOST data (bounds, counts, sums: a few hundred bytes per rank that
// the stage before has just synchronised onto the host).  Through the GPU and back each would be
// a pinned H2D, ncclAllGather, D2H and stream sync, three per reduce.  All ranks of this engine's scope live on one node, so they meet in a POSIX
// shared-memory segment instead: rank p writes its vector into slot p of a double-buffered
// mailbox and publishes a sequence number with release semantics; everybody spins (acquire) until
// all R slots carry the current number.  A few microseconds, no GPU work, no stream sync.
// Set up once per context by two NCCL all-gathers (token + host check, then "opened"); ranks on
// different hosts, or a failed shm_open, keep the NCCL path.
constexpr int MB_DOUBLES = 192;
struct MboxSlot {
  std::atomic<u64> seq[2];
  double data[2][MB_DOUBLES];
};
static_assert(sizeof(std::atomic<u64>) == 8, "lock-free 64-bit atomics");

u64 host_hash() {
  char name[256];
  memset(name, 0, sizeof(name));
  gethostname(name, sizeof(name) - 1);
  u64 h = 1469598103934665603ull;
  for (const char* p = name; *p; ++p) { h ^= (unsigned char)*p; h *= 1099511628211ull; }
  return h & ((1ull << 52) - 1);  // travels as a double
}

int ensure_ws(tml_ctx* c, RunWs** out) {
  void** slot = tml_run_ws_slot_(c);
  if (!*slot) {
    RunWs* w = new RunWs();
    CKC(cudaMalloc(&w->d_send, XV * sizeof(double)));
    CKC(cudaMalloc(&w->d_recv, (size_t)TML_MAX_RANKS * XV * sizeof(double)));
    CKC(cudaHostAlloc(&w->h_send, XV * sizeof(double), cudaHostAllocDefault));
    CKC(cudaHostAlloc(&w->h_recv, (size_t)TML_MAX_RANKS * XV * sizeof(double), cudaHostAllocDefault));
    CKC(cudaStreamCreateWithFlags(&w->side, cudaStreamNonBlocking));
    CKC(cudaEventCreateWithFlags(&w->side_gate, cudaEventDisableTiming));
    *slot = w;
  }
  *out = (RunWs*)*slot;
  return TML_OK;
}

template <typename T>
int grow(T** p, u64* cap, u64 need) {
  if (need <= *cap && *p) return TML_OK;
  if (*p) { cudaFree(*p); *p = nullptr; *cap = 0; }
  u64 n = need + need / 4 + 64;
  CKC(cudaMalloc(p, (size_t)n * sizeof(T)));
  *cap = n;
  return TML_OK;
}

struct Run {
  tml_ctx* c;
  RunWs* w;
  const tml_comm* comm;
  cudaStream_t s;
  int rank, world;
  u32 n_exchanges = 0;

  int nccl_gather(const double* vec, int len, double* all) {
    memcpy(w->h_send, vec, (size_t)len * sizeof(double));
    CKC(cudaMemcpyAsync(w->d_send, w->h_send, (size_t)len * sizeof(double), cudaMemcpyHostToDevice, s));
    CKN(g_nccl.AllGather(w->d_send, w->d_recv, (size_t)len, ncclDouble, (ncclComm_t)comm->nccl_comm, s));
    CKC(cudaMemcpyAsync(w->h_recv, w->d_recv, (size_t)len * world * sizeof(double), cudaMemcpyDeviceToHost, s));
    CKC(cudaStreamSynchronize(s));
    memcpy(all, w->h_recv, (size_t)len * world * sizeof(double));
    return TML_OK;
  }

  // once per context: agree on a shared-memory mailbox (all ranks on one host), else stay on NCCL
  int mbox_setup() {
    w->mbox_tried = true;
    const char* off = getenv("TML_NO_MAILBOX");
    const bool disabled = off && off[0] == '1';
    double mine[4] = {(double)host_hash(), (double)getpid(), 0.0, disabled ? 1.0 : 0.0};
    if (rank == 0) {
      u64 t = (u64)std::chrono::steady_clock::now().time_since_epoch().count();
      mine[2] = (double)((t ^ ((u64)getpid() << 20)) & ((1ull << 50) - 1));
    }
    std::vector<double> all((size_t)world * 4);
    CKT(nccl_gather(mine, 4, all.data()));
    bool same = true;
    for (int p = 0; p < world; ++p) same = same && all[(size_t)p * 4] == all[0] && all[(size_t)p * 4 + 3] == 0.0;
    char name[96];
    snprintf(name, sizeof(name), "/tml_b200_%llu_%llu", (unsigned long long)all[1], (unsigned long long)all[2]);
    const size_t bytes = sizeof(MboxSlot) * (size_t)world;
    void* mem = nullptr;
    int fd = -1;
    if (same && rank == 0) {
      fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
      if (fd >= 0 && ftruncate(fd, (off_t)bytes) == 0) {
        mem = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        if (mem == MAP_FAILED) mem = nullptr;
        else memset(mem, 0, bytes);
      }
    }
    double ok1[1] = {(!same || rank != 0 || mem) ? 1.0 : 0.0};
    std::vector<double> oks((size_t)world);
    CKT(nccl_gather(ok1, 1, oks.data()));  // rank 0 has created the segment (or given up)
    bool go = same && oks[0] == 1.0;
    if (go && rank != 0) {
      fd = shm_open(name, O_RDWR, 0600);
      if (fd >= 0) {
        mem = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        if (mem == MAP_FAILED) mem = nullptr;
      }
    }
    if (fd >= 0) close(fd);
    double ok2[1] = {(!go || mem) ? 1.0 : 0.0};
    CKT(nccl_gather(ok2, 1, oks.data()));  // everybody has mapped it: the name can go
    if (rank == 0 && same) shm_unlink(name);
    for (int p = 0; p < world; ++p) go = go && oks[p] == 1.0;
    if (go && mem) { w->mbox = mem; w->mbox_bytes = bytes; w->mbox_seq = 0; }
    else if (mem) munmap(mem, bytes);
    return TML_OK;
  }

  int mbox_gather(const double* vec, int len, double* all) {
    MboxSlot* slots = (MboxSlot*)w->mbox;
    const u64 seq = ++w->mbox_seq;
    const int b = (int)(seq & 1ull);
    memcpy(slots[rank].data[b], vec, (size_t)len * sizeof(double));
    slots[rank].seq[b].store(seq, std::memory_order_release);
    const auto t0 = std::chrono::steady_clock::now();
    for (int p = 0; p < world; ++p) {
      unsigned spins = 0;
      while (slots[p].seq[b].load(std::memory_order_acquire) < seq) {
        if ((++spins & 0xfffu) == 0u) {
          if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(60))
            return tml_set_error_(TML_ERR_STATE, "mailbox exchange %llu: rank %d never arrived", (unsigned long long)seq, p);
          sched_yield();
        }
      }
      memcpy(all + (size_t)p * len, slots[p].data[b], (size_t)len * sizeof(double));
    }
    return TML_OK;
  }

  // one small exchange: every rank contributes `len` doubles; all[r * len + i]
  int xchg(const double* vec, int len, double* all) {
    ++n_exchanges;
    if (world == 1) { memcpy(all, vec, (size_t)len * sizeof(double)); return TML_OK; }
    if (len > XV) return tml_set_error_(TML_ERR_ARG, "exchange vector too long (%d)", len);
    if (!w->mbox_tried) CKT(mbox_setup());
    if (w->mbox && len <= MB_DOUBLES) return mbox_gather(vec, len, all);
    memcpy(w->h_send, vec, (size_t)len * sizeof(double));
    CKC(cudaMemcpyAsync(w->d_send, w->h_send, (size_t)len * sizeof(double), cudaMemcpyHostToDevice, s));
    CKN(g_nccl.AllGather(w->d_send, w->d_recv, (size_t)len, ncclDouble, (ncclComm_t)comm->nccl_comm, s));
    CKC(cudaMemcpyAsync(w->h_recv, w->d_recv, (size_t)len * world * sizeof(double), cudaMemcpyDeviceToHost, s));
    CKC(cudaStreamSynchronize(s));
    memcpy(all, w->h_recv, (size_t)len * world * sizeof(double));
    return TML_OK;
  }
};

// ------------------------------------------------------------------ packing
constexpr int INFO_LEN = 23, PROC_LEN = 17, ALIGN_LEN = 15, HANDLE_LEN = 9;  // 72-byte handle = 9 doubles

void pack_info(const tml_win_info& i, double* v) {
  int k = 0;
  v[k++] = (double)i.n_retained; v[k++] = (double)i.latest_step; v[k++] = (double)i.monotone;
  v[k++] = (double)i.dup_rows;
  for (int q = 0; q < 2; ++q) v[k++] = (double)i.n_rows[q];
  for (int q = 0; q < 2; ++q) v[k++] = (double)i.n_cand[q];
  for (int q = 0; q < 2; ++q) v[k++] = (double)i.lo[q];   // step ids < 2^53
  for (int q = 0; q < 2; ++q) v[k++] = (double)i.hi[q];
  for (int q = 0; q < 7; ++q) v[k++] = i.t_sums[q];
  v[k++] = (double)i.t_count; v[k++] = (double)i.n_both;
  for (int q = 0; q < 2; ++q) v[k++] = (double)i.dense[q];
}
void unpack_info(const double* v, tml_win_info* i) {
  memset(i, 0, sizeof(*i));
  int k = 0;
  i->n_retained = (u64)llround(v[k++]); i->latest_step = (u64)llround(v[k++]);
  i->monotone = (u32)llround(v[k++]); i->dup_rows = (u32)llround(v[k++]);
  for (int q = 0; q < 2; ++q) i->n_rows[q] = (u64)llround(v[k++]);
  for (int q = 0; q < 2; ++q) i->n_cand[q] = (u64)llround(v[k++]);
  for (int q = 0; q < 2; ++q) i->lo[q] = (u64)llround(v[k++]);
  for (int q = 0; q < 2; ++q) i->hi[q] = (u64)llround(v[k++]);
  for (int q = 0; q < 7; ++q) i->t_sums[q] = v[k++];
  i->t_count = (u64)llround(v[k++]); i->n_both = (u64)llround(v[k++]);
  for (int q = 0; q < 2; ++q) i->dense[q] = (u32)llround(v[k++]);
}
void pack_proc(const tml_proc_agg& a, double* v) {
  int k = 0;
  v[k++] = (double)a.n; v[k++] = (double)a.n_gpu; v[k++] = a.ts_min; v[k++] = a.ts_max;
  v[k++] = a.sum_cpu; v[k++] = a.max_cpu; v[k++] = a.sum_rss; v[k++] = a.max_rss;
  v[k++] = a.sum_used; v[k++] = a.max_used; v[k++] = a.sum_resv; v[k++] = a.max_resv;
  v[k++] = a.max_total; v[k++] = a.max_ratio; v[k++] = (double)a.max_cores;
  v[k++] = (double)a.any_gpu_available; v[k++] = a.sum_cpu_lo;
}
void unpack_proc(const double* v, tml_proc_agg* a) {
  memset(a, 0, sizeof(*a));
  int k = 0;
  a->n = (u64)llround(v[k++]); a->n_gpu = (u64)llround(v[k++]); a->ts_min = v[k++]; a->ts_max = v[k++];
  a->sum_cpu = v[k++]; a->max_cpu = v[k++]; a->sum_rss = v[k++]; a->max_rss = v[k++];
  a->sum_used = v[k++]; a->max_used = v[k++]; a->sum_resv = v[k++]; a->max_resv = v[k++];
  a->max_total = v[k++]; a->max_ratio = v[k++]; a->max_cores = (u32)llround(v[k++]);
  a->any_gpu_available = (u32)llround(v[k++]); a->sum_cpu_lo = v[k++];
}
void pack_align(const tml_align_info& a, double* v) {
  v[0] = (double)a.n_common; v[1] = (double)a.start_step; v[2] = (double)a.end_step; v[3] = (double)a.n_rows;
  for (int q = 0; q < 7; ++q) v[4 + q] = a.t_sums[q];
  for (int q = 0; q < 4; ++q) v[11 + q] = a.m_sums[q];
}

struct Aligned {  // one rank's block of an alignment exchange
  u64 n_common, start, end, n_rows;
  double t_sums[7], m_sums[4];
  unsigned char handle[72];
};
void unpack_align(const double* v, bool handles, Aligned* a) {
  a->n_common = (u64)llround(v[0]); a->start = (u64)llround(v[1]); a->end = (u64)llround(v[2]);
  a->n_rows = (u64)llround(v[3]);
  memcpy(a->t_sums, v + 4, sizeof(a->t_sums));
  memcpy(a->m_sums, v + 11, sizeof(a->m_sums));
  if (handles) memcpy(a->handle, v + ALIGN_LEN, 72); else memset(a->handle, 0, 72);
}

// ------------------------------------------------------------------ trend band layout
// analytics/trends/core.py:38-84 + schema.py:27-62, as traceml_b200/reduce.py:trend_layout
bool trend_layout(u64 n, u64 min_points, double warmup_frac, u64 lo[3], u64 hi[3]) {
  static const double BANDS[3][2] = {{0.15, 0.25}, {0.45, 0.55}, {0.90, 1.00}};
  if (n < min_points) return false;
  const u64 length = n < 10000 ? n : 10000;
  if (length < min_points) return false;
  const u64 off = n - length;
  const u64 warm = (u64)std::floor((double)length * warmup_frac);
  const u64 stable = length - warm;
  if (stable < min_points) return false;
  for (int b = 0; b < 3; ++b) {
    long long st = (long long)std::floor((double)stable * BANDS[b][0]);
    long long en = (long long)std::ceil((double)stable * BANDS[b][1]);
    const long long nn = (long long)stable;
    st = st < 0 ? 0 : (st > nn - 1 ? nn - 1 : st);
    if (en > nn) en = nn;
    if (en < st + 1) en = st + 1;
    lo[b] = off + warm + (u64)st;
    hi[b] = off + warm + (u64)en;
  }
  return true;
}

// ------------------------------------------------------------------ the run
constexpr u64 TML_FUSED_MIN_ROWS = 1u << 17;  // == TML_EXACT_SUM_MAX: below it the staged path gives reference-order sums
constexpr u64 P2P_MIN_ROWS = 1000000;  // reduce.py: the one-shot IPC mapping pays above this

struct KindState {
  tml_kind_result* res;
  std::vector<Aligned> blocks;  // by global rank (valid for ranks in res->used)
  bool from_spec = false;       // aligned window == every rank's own window: aligned sums are window sums
};

u32 mode_for(const Run& r, u32 exchange, u64 n_common) {
  if (r.world == 1) return TML_XCHG_LOCAL;
  if (exchange == TML_XCHG_P2P || exchange == TML_XCHG_A2A) return exchange;
  if (n_common < P2P_MIN_ROWS && !r.w->p2p_warm) return TML_XCHG_A2A;
  return TML_XCHG_P2P;
}

int parse_aligns(Run& r, const double* all, int stride, int off, bool handles, u32 kind,
                 const tml_win_info* infos, const std::vector<int>& part, KindState* ks) {
  tml_kind_result* res = ks->res;
  ks->blocks.assign(r.world, Aligned());
  u64 n_common = 0;
  for (int p = 0; p < r.world; ++p) {
    unpack_align(all + (size_t)p * stride + off, handles, &ks->blocks[p]);
    if (ks->blocks[p].n_common > n_common) n_common = ks->blocks[p].n_common;
  }
  res->n_common = n_common;
  if (n_common == 0) return TML_OK;
  for (int p : part) {
    const Aligned& a = ks->blocks[p];
    if (a.n_rows == 0) continue;
    const u32 i = res->n_used++;
    res->used[i] = p;
    res->n_rows[i] = a.n_rows;
    memcpy(res->t_sums[i], a.t_sums, sizeof(a.t_sums));
    memcpy(res->m_sums[i], a.m_sums, sizeof(a.m_sums));
    res->start_step = a.start; res->end_step = a.end;
  }
  (void)kind; (void)infos;
  return TML_OK;
}

int export_block(Run& r, u32 kind, u32 exchange, const tml_align_info& a, bool handles, double* v) {
  pack_align(a, v);
  if (handles) {
    memset(v + ALIGN_LEN, 0, HANDLE_LEN * sizeof(double));
    if (mode_for(r, exchange, a.n_common) == TML_XCHG_P2P && a.n_rows > 0) {
      unsigned char h[72];
      uint64_t off = 0;
      CKT(tml_win_rows_export(r.c, kind, h, &off));
      memcpy(h + 64, &off, 8);
      memcpy(v + ALIGN_LEN, h, 72);
    }
  }
  return TML_OK;
}

int align_kind(Run& r, u32 kind, u32 window, u32 exchange, const tml_win_info* infos, const double* spec_all,
               int spec_stride, int spec_off, bool spec_handles, KindState* ks) {
  tml_kind_result* res = ks->res;
  std::vector<int> part;
  for (int p = 0; p < r.world; ++p) if (infos[p].n_cand[kind] > 0) part.push_back(p);
  res->observed = (u32)part.size();
  if (part.empty()) return TML_OK;
  u64 glo = 0, ghi = ~0ull;
  bool all_dense = true;
  for (int p : part) {
    if (infos[p].lo[kind] > glo) glo = infos[p].lo[kind];
    if (infos[p].hi[kind] < ghi) ghi = infos[p].hi[kind];
    all_dense = all_dense && infos[p].dense[kind] != 0;
  }
  if (ghi < glo) return TML_OK;
  const u64 span = ghi - glo + 1;
  const bool handles = r.world > 1 && exchange != TML_XCHG_A2A;  // layout of a non-speculative block
  const int alen = ALIGN_LEN + (handles ? HANDLE_LEN : 0);
  std::vector<double> all((size_t)r.world * alen), mine(alen, 0.0);
  tml_align_info a;
  if (all_dense) {
    bool same_window = spec_all != nullptr && span <= window;
    for (int p : part) same_window = same_window && infos[p].lo[kind] == glo && infos[p].hi[kind] == ghi;
    if (same_window) {  // every participant speculated on exactly [glo, ghi]
      ks->from_spec = true;
      return parse_aligns(r, spec_all, spec_stride, spec_off, spec_handles, kind, infos, part, ks);
    }
    const u64 n_common = span < window ? span : window;
    CKT(tml_win_select_dense(r.c, kind, ghi - n_common + 1, n_common, r.s, &a));
  } else {
    CKT(grow(&r.w->d_presence, &r.w->cap_presence, span));
    CKT(tml_win_presence(r.c, kind, glo, span, r.w->d_presence, r.s));
    if (r.world > 1)
      CKN(g_nccl.AllReduce(r.w->d_presence, r.w->d_presence, (size_t)span, ncclUint8, ncclMin,
                           (ncclComm_t)r.comm->nccl_comm, r.s));
    CKT(tml_win_select(r.c, kind, glo, span, r.w->d_presence, window, r.s, &a));
  }
  CKT(export_block(r, kind, exchange, a, handles, mine.data()));
  CKT(r.xchg(mine.data(), alen, all.data()));
  return parse_aligns(r, all.data(), alen, 0, handles, kind, infos, part, ks);
}

int reduce_pass(Run& r, u32 kind, u32 mask, u32 mode, KindState* ks, int series_slot) {
  tml_kind_result* res = ks->res;
  const u64 n = res->n_common;
  RunWs* w = r.w;
  CKT(grow(&w->d_series[series_slot], &w->cap_series[series_slot], (u64)TML_SERIES_PER_STEP * n));
  res->series = w->d_series[series_slot];
  const int W = r.world, g = r.rank;
  const u64 lo = (n * (u64)g) / (u64)W, hi = (n * (u64)(g + 1)) / (u64)W;
  res->shard_lo = lo; res->shard_hi = hi;
  bool mine_used = false;
  for (u32 i = 0; i < res->n_used; ++i) mine_used = mine_used || res->used[i] == g;
  tml_reduce_args ra;
  memset(&ra, 0, sizeof(ra));
  ra.n_ranks = res->n_used; ra.mask = mask; ra.n_common = n; ra.shard_lo = lo; ra.shard_hi = hi;
  ra.series = w->d_series[series_slot];
  if (mode == TML_XCHG_LOCAL) {
    ra.rows[0] = tml_win_rows(r.c, kind);
  } else if (mode == TML_XCHG_A2A) {
    // step-sharded send/recv: I receive rows [lo, hi) of every rank, ((R-1)/R) n 64 B in all;
    // K4 addresses them through virtual bases (row j of rank p at recv[p] + (j - lo) * 64)
    const u64 my_len = hi - lo;
    CKT(grow(&w->d_recv_rows, &w->cap_recv_rows, (u64)W * my_len * 64 + 64));
    const char* src = (const char*)tml_win_rows(r.c, kind);
    if (!mine_used || !src) {
      CKT(grow(&w->d_zero_rows, &w->cap_zero_rows, n * 64 + 64));
      CKC(cudaMemsetAsync(w->d_zero_rows, 0, (size_t)n * 64, r.s));
      src = w->d_zero_rows;
    }
    CKN(g_nccl.GroupStart());
    for (int d = 0; d < W; ++d) {
      const u64 dlo = (n * (u64)d) / (u64)W, dhi = (n * (u64)(d + 1)) / (u64)W;
      if (dhi > dlo)
        CKN(g_nccl.Send(src + dlo * 64, (size_t)(dhi - dlo) * 8, ncclDouble, d, (ncclComm_t)r.comm->nccl_comm, r.s));
      if (my_len)
        CKN(g_nccl.Recv(w->d_recv_rows + (u64)d * my_len * 64, (size_t)my_len * 8, ncclDouble, d,
                        (ncclComm_t)r.comm->nccl_comm, r.s));
    }
    CKN(g_nccl.GroupEnd());
    for (u32 i = 0; i < res->n_used; ++i) {
      const long long off = ((long long)res->used[i] * (long long)my_len - (long long)lo) * 64;
      ra.rows[i] = w->d_recv_rows + off;
    }
  } else {  // peer loads fused into K4 (no barrier needed: see reduce.py:_reduce_pass)
    for (u32 i = 0; i < res->n_used; ++i) {
      const int p = res->used[i];
      if (p == g) { ra.rows[i] = tml_win_rows(r.c, kind); continue; }
      void* base = nullptr;
      CKT(tml_peer_open(r.c, ks->blocks[p].handle, &base));
      u64 off = 0;
      memcpy(&off, ks->blocks[p].handle + 64, 8);
      ra.rows[i] = (const char*)base + off;
    }
    w->p2p_warm = true;
  }
  if (hi > lo) CKT(tml_win_reduce(r.c, &ra, r.s));
  return TML_OK;
}

// `extra` (n_extra doubles per rank, may be 0) rides in the band exchange: the deferred
// reference-order sums of K3e, so that they cost no exchange of their own.  *extra_done tells the
// caller whether the exchange happened (no aligned window -> no band exchange).
int bands(Run& r, tml_kind_result* res, const double* extra = nullptr, int n_extra = 0,
          double* extra_all = nullptr, bool* extra_done = nullptr) {
  const u64 n = res->n_common;
  if (extra_done) *extra_done = false;
  if (n == 0 || !res->series) return TML_OK;
  tml_band_args a;
  memset(&a, 0, sizeof(a));
  a.n_common = n; a.shard_lo = res->shard_lo; a.shard_hi = res->shard_hi;
  u64 lo[3], hi[3];
  if (trend_layout(n, 200, 0.10, lo, hi)) for (int b = 0; b < 3; ++b) { a.band_lo[0][b] = lo[b]; a.band_hi[0][b] = hi[b]; }
  if (trend_layout(n, 50, 0.0, lo, hi)) for (int b = 0; b < 3; ++b) { a.band_lo[1][b] = lo[b]; a.band_hi[1][b] = hi[b]; }
  a.tail_first[0] = 0;
  a.tail_first[1] = n - (n < 1000 ? n : 1000);
  tml_band_out bo;
  CKT(tml_win_bands(r.c, res->series, &a, r.s, &bo));
  double vec[128 + 16];
  for (int s = 0; s < 16; ++s)
    for (int b = 0; b < 3; ++b) { vec[s * 3 + b] = bo.sum[s][b]; vec[48 + s * 3 + b] = (double)bo.cnt[s][b]; }
  for (int s = 0; s < 16; ++s) { vec[96 + s] = bo.tail_first[s]; vec[112 + s] = bo.tail_last[s]; }
  const int BL = 128 + (n_extra > 0 && n_extra <= 16 ? n_extra : 0);
  for (int q = 128; q < BL; ++q) vec[q] = extra[q - 128];
  std::vector<double> all((size_t)r.world * BL);
  CKT(r.xchg(vec, BL, all.data()));
  if (BL > 128 && extra_all) {
    for (int p = 0; p < r.world; ++p) memcpy(extra_all + (size_t)p * n_extra, all.data() + (size_t)p * BL + 128, n_extra * sizeof(double));
    if (extra_done) *extra_done = true;
  }
  for (int s = 0; s < 16; ++s) {
    for (int b = 0; b < 3; ++b) {
      double acc = 0.0;  // rank order, like reduce.py's sum()
      u64 cnt = 0;
      for (int p = 0; p < r.world; ++p) {
        acc += all[(size_t)p * BL + s * 3 + b];
        cnt += (u64)llround(all[(size_t)p * BL + 48 + s * 3 + b]);
      }
      res->band_sum[s][b] = acc;
      res->band_cnt[s][b] = cnt;
    }
    double tf = NAN, tl = NAN;
    for (int p = 0; p < r.world && std::isnan(tf); ++p) tf = all[(size_t)p * BL + 96 + s];
    for (int p = 0; p < r.world && std::isnan(tl); ++p) tl = all[(size_t)p * BL + 112 + s];
    res->tail_first[s] = tf;
    res->tail_last[s] = tl;
  }
  res->has_bands = 1;
  return TML_OK;
}

double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

}  // namespace

extern "C" int tml_reduce_run(tml_ctx* c, const tml_comm* comm, const tml_reduce_run_args* args, void* stream,
                              tml_reduce_run_out* out) {
  if (!c || !args || !out || args->window == 0) return TML_ERR_ARG;
  const int world = comm ? comm->world : 1, rank = comm ? comm->rank : 0;
  if (world < 1 || world > (int)TML_MAX_RANKS || rank < 0 || rank >= world) return TML_ERR_ARG;
  if (world > 1) {
    if (!comm->nccl_comm) return tml_set_error_(TML_ERR_ARG, "world > 1 needs an NCCL communicator");
    std::call_once(g_nccl_once, load_nccl);
    if (!g_nccl.ok) return tml_set_error_(TML_ERR_UNSUPPORTED, "libnccl.so.2 is not loadable in this process");
  }
  const u32 window = args->window;
  const u32 exchange = args->exchange;
  if (exchange > TML_XCHG_A2A) return TML_ERR_ARG;
  memset(out, 0, sizeof(*out));
  Run r;
  r.c = c; r.comm = comm; r.s = (cudaStream_t)stream; r.rank = rank; r.world = world;
  CKT(ensure_ws(c, &r.w));
  const double t0 = now_ms();

  // ---- stage 1: local window + bounds; process aggregates and the speculative alignment ride along
  // K6 on the side stream: three tiny kernels that would otherwise sit in front of K3a;
  // tml_proc_reduce_collect waits on their own event
  if (args->proc_rows) {
    CKC(cudaEventRecord(r.w->side_gate, r.s));
    CKC(cudaStreamWaitEvent(r.w->side, r.w->side_gate, 0));
    CKT(tml_proc_reduce_launch(c, args->proc_rows, r.w->side));
  }
  // ---- single rank, bulk window: ring -> series in ONE pass (k_window_fused); the WindowRows
  // that K3a would write for K4 to re-read never exist.  Falls through to the staged path when the
  // window is not dense (re-flushed step ids, rows without memory, ...).
  if (world == 1) {
    u64 n_ret = 0, n_win = 0;
    CKT(tml_win_peek(c, window, &n_ret, &n_win));
    if (n_win > (u64)TML_FUSED_MIN_ROWS) {
      CKT(grow(&r.w->d_series[0], &r.w->cap_series[0], (u64)TML_SERIES_PER_STEP * n_win));
      tml_win_info finfo;
      tml_align_info fal;
      uint32_t ok = 0;
      CKT(tml_win_fused(c, window, r.w->d_series[0], r.s, &finfo, &fal, &ok));
      if (ok) {
        tml_proc_agg pagg0;
        memset(&pagg0, 0, sizeof(pagg0));
        if (args->proc_rows) CKT(tml_proc_reduce_collect(c, &pagg0));
        out->n_ranks = 1;
        out->infos[0] = finfo;
        out->procs[0] = pagg0;
        for (tml_kind_result* res : {&out->time, &out->mem}) {
          res->observed = 1; res->n_used = 1; res->used[0] = 0;
          res->n_common = fal.n_common; res->start_step = fal.start_step; res->end_step = fal.end_step;
          res->n_rows[0] = fal.n_rows;
          memcpy(res->t_sums[0], fal.t_sums, sizeof(fal.t_sums));
          memcpy(res->m_sums[0], fal.m_sums, sizeof(fal.m_sums));
          res->series = r.w->d_series[0];
          res->shard_lo = 0; res->shard_hi = fal.n_common;
        }
        out->exchange_used = TML_XCHG_LOCAL;
        out->fused_pass = 2;  // 2: K3a and K4 fused as well (no WindowRows)
        const double tf = now_ms();
        CKT(bands(r, &out->time));
        memcpy(out->mem.band_sum, out->time.band_sum, sizeof(out->time.band_sum));
        memcpy(out->mem.band_cnt, out->time.band_cnt, sizeof(out->time.band_cnt));
        memcpy(out->mem.tail_first, out->time.tail_first, sizeof(out->time.tail_first));
        memcpy(out->mem.tail_last, out->time.tail_last, sizeof(out->time.tail_last));
        out->mem.has_bands = out->time.has_bands;
        const double te = now_ms();
        out->n_exchanges = r.n_exchanges;
        out->k3a_ms = finfo.kernel_ms;
        out->k4_ms = 0.0;
        out->stage_ms[0] = tf - t0; out->stage_ms[1] = 0.0; out->stage_ms[2] = 0.0;
        out->stage_ms[3] = te - tf; out->stage_ms[4] = te - t0;
        return TML_OK;
      }
    }
  }
  tml_win_info info;
  // R > 1: K3e (reference-order sums) runs beside the exchanges and K4; its result is collected
  // in stage 5 and rides in the band exchange
  const bool deferred = world > 1;
  tml_win_set_defer(c, deferred ? 1 : 0);
  const int prc = tml_win_prepare(c, window, r.s, &info);
  tml_win_set_defer(c, 0);
  CKT(prc);
  tml_proc_agg pagg;
  memset(&pagg, 0, sizeof(pagg));
  if (args->proc_rows) CKT(tml_proc_reduce_collect(c, &pagg));
  // Memory candidate limit (step_memory/loader.py:215): only the newest max(20 W, W + 1)
  // distinct step ids of a rank enter the memory alignment.  The ring normally holds 1.5 W
  // rows, so this binds only for a small window over a long ring; the rank then advertises
  // the step id of its limit-th newest candidate as its lower bound, and every later stage
  // works on [max lo, min hi] without ever seeing the older candidates.
  {
    const u64 limit = (u64)window * 20ull > (u64)window + 1ull ? (u64)window * 20ull : (u64)window + 1ull;
    if (info.n_cand[TML_KIND_MEM] > limit) {
      u64 thr;
      if (info.dense[TML_KIND_MEM]) {
        thr = info.hi[TML_KIND_MEM] - limit + 1;  // consecutive ids
      } else {  // holes / re-flushed ids: select the newest `limit` of the rank's own candidates
        const u64 lo = info.lo[TML_KIND_MEM], span = info.hi[TML_KIND_MEM] - lo + 1;
        CKT(grow(&r.w->d_presence, &r.w->cap_presence, span));
        CKT(tml_win_presence(c, TML_KIND_MEM, lo, span, r.w->d_presence, r.s));
        tml_align_info own;
        CKT(tml_win_select(c, TML_KIND_MEM, lo, span, r.w->d_presence, (uint32_t)limit, r.s, &own));
        thr = own.start_step;
      }
      info.lo[TML_KIND_MEM] = thr;
      info.n_cand[TML_KIND_MEM] = limit;
    }
  }
  const bool spec_handles = world > 1 && exchange != TML_XCHG_A2A;
  const int plen = args->proc_rows ? PROC_LEN : 0;
  const int slen = args->speculate ? ALIGN_LEN + (spec_handles ? HANDLE_LEN : 0) : 0;
  const int per = INFO_LEN + plen + slen;
  std::vector<double> mine(per, 0.0), all((size_t)world * per);
  pack_info(info, mine.data());
  if (plen) pack_proc(pagg, mine.data() + INFO_LEN);
  if (slen && info.dense[TML_KIND_TIME] && info.n_cand[TML_KIND_TIME] > 0) {
    tml_align_info a;
    CKT(tml_win_select_dense(c, TML_KIND_TIME, info.lo[TML_KIND_TIME], info.n_cand[TML_KIND_TIME], r.s, &a));
    CKT(export_block(r, TML_KIND_TIME, exchange, a, spec_handles, mine.data() + INFO_LEN + plen));
  }
  CKT(r.xchg(mine.data(), per, all.data()));
  out->n_ranks = (u32)world;
  for (int p = 0; p < world; ++p) {
    unpack_info(all.data() + (size_t)p * per, &out->infos[p]);
    if (plen) unpack_proc(all.data() + (size_t)p * per + INFO_LEN, &out->procs[p]);
  }
  out->infos[rank].kernel_ms = info.kernel_ms;
  const double t1 = now_ms();

  // ---- stages 2-3: alignment (one for both sections when the candidate rows coincide)
  bool merged = true;
  for (int p = 0; p < world; ++p) {
    const tml_win_info& i = out->infos[p];
    merged = merged && i.n_cand[0] == i.n_cand[1] && i.n_cand[1] == i.n_both;
  }
  KindState kt, km;
  kt.res = &out->time; km.res = &out->mem;
  CKT(align_kind(r, TML_KIND_TIME, window, exchange, out->infos, slen ? all.data() : nullptr, per,
                 INFO_LEN + plen, spec_handles, &kt));
  if (merged) {
    const tml_kind_result& t = out->time;
    tml_kind_result& m = out->mem;
    m.observed = t.observed; m.n_used = t.n_used; m.n_common = t.n_common;
    m.start_step = t.start_step; m.end_step = t.end_step;
    memcpy(m.used, t.used, sizeof(t.used));
    memcpy(m.n_rows, t.n_rows, sizeof(t.n_rows));
    memcpy(m.t_sums, t.t_sums, sizeof(t.t_sums));
    memcpy(m.m_sums, t.m_sums, sizeof(t.m_sums));
    km.blocks = kt.blocks;
  } else {
    CKT(align_kind(r, TML_KIND_MEM, window, exchange, out->infos, nullptr, 0, 0, false, &km));
  }
  const double t2 = now_ms();

  // ---- stage 4: row exchange + per-step reduce
  const tml_kind_result& t = out->time;
  const tml_kind_result& m = out->mem;
  bool same = t.n_common > 0 && t.n_common == m.n_common && t.start_step == m.start_step &&
              t.end_step == m.end_step && t.n_used == m.n_used;
  for (u32 i = 0; same && i < t.n_used; ++i) same = t.used[i] == m.used[i];
  const u32 mode = mode_for(r, exchange, t.n_common ? t.n_common : m.n_common);
  out->exchange_used = mode;
  out->fused_pass = same ? 1u : 0u;
  if (same) {
    CKT(reduce_pass(r, TML_KIND_TIME, TML_MASK_TIME | TML_MASK_MEM, mode, &kt, 0));
    out->mem.series = out->time.series;
    out->mem.shard_lo = out->time.shard_lo; out->mem.shard_hi = out->time.shard_hi;
  } else {
    if (t.n_common && t.n_used) CKT(reduce_pass(r, TML_KIND_TIME, TML_MASK_TIME, mode_for(r, exchange, t.n_common), &kt, 0));
    if (m.n_common && m.n_used) CKT(reduce_pass(r, TML_KIND_MEM, TML_MASK_MEM, mode_for(r, exchange, m.n_common), &km, 1));
  }
  const double t3 = now_ms();

  // ---- stage 5: trend bands (+ the deferred reference-order sums of every rank)
  double exact_mine[7] = {0}, exact_all[TML_MAX_RANKS * 7];
  bool exact_done = false;
  if (deferred) CKT(tml_win_exact_collect(c, r.s, exact_mine));
  CKT(bands(r, &out->time, deferred ? exact_mine : nullptr, deferred ? 7 : 0, exact_all, &exact_done));
  if (same) {
    memcpy(out->mem.band_sum, out->time.band_sum, sizeof(out->time.band_sum));
    memcpy(out->mem.band_cnt, out->time.band_cnt, sizeof(out->time.band_cnt));
    memcpy(out->mem.tail_first, out->time.tail_first, sizeof(out->time.tail_first));
    memcpy(out->mem.tail_last, out->time.tail_last, sizeof(out->time.tail_last));
    out->mem.has_bands = out->time.has_bands;
  } else {
    CKT(bands(r, &out->mem));
  }
  if (deferred) {
    if (!exact_done) CKT(r.xchg(exact_mine, 7, exact_all));  // no aligned window: no band exchange to ride in
    for (int p = 0; p < world; ++p) memcpy(out->infos[p].t_sums, exact_all + (size_t)p * 7, 7 * sizeof(double));
    // lock step: the aligned window IS each rank's window, so its sums are the window sums with
    // avg_step_cpu := traced (alignment.py:72); otherwise tml_win_select* computed exact aligned sums
    tml_kind_result* both[2] = {&out->time, merged ? &out->mem : nullptr};
    if (kt.from_spec) {
      for (tml_kind_result* res : both) {
        if (!res) continue;
        for (u32 i = 0; i < res->n_used; ++i) {
          const double* e = exact_all + (size_t)res->used[i] * 7;
          memcpy(res->t_sums[i], e, 7 * sizeof(double));
          res->t_sums[i][4] = e[5];
        }
      }
    }
  }
  const double t4 = now_ms();
  out->n_exchanges = r.n_exchanges;
  out->k3a_ms = info.kernel_ms;
  out->k4_ms = tml_kernel_ms(c, 1);
  {
    // TML_TIMELINE=1: device timeline of this reduce on stderr (rank 0), ms since K3a began
    static const bool tl = [] { const char* e = getenv("TML_TIMELINE"); return e && e[0] == '1'; }();
    if (tl && r.rank == 0)
      fprintf(stderr, "[tml timeline] k3a_end %.3f k4_launch %.3f k3e_end %.3f k4_end %.3f | host prepare %.3f "
              "align %.3f reduce %.3f bands %.3f\n", info.kernel_ms, tml_kernel_ms(c, 2), tml_kernel_ms(c, 3),
              tml_kernel_ms(c, 4), t1 - t0, t2 - t1, t3 - t2, t4 - t3);
  }
  out->stage_ms[0] = t1 - t0; out->stage_ms[1] = t2 - t1; out->stage_ms[2] = t3 - t2;
  out->stage_ms[3] = t4 - t3; out->stage_ms[4] = t4 - t0;
  return TML_OK;
}

extern "C" void tml_run_ws_free_(void* p) {
  RunWs* w = (RunWs*)p;
  if (!w) return;
  cudaFree(w->d_send); cudaFree(w->d_recv); cudaFreeHost(w->h_send); cudaFreeHost(w->h_recv);
  cudaFree(w->d_presence); cudaFree(w->d_series[0]); cudaFree(w->d_series[1]);
  cudaFree(w->d_recv_rows); cudaFree(w->d_zero_rows);
  if (w->mbox) munmap(w->mbox, w->mbox_bytes);
  if (w->side) cudaStreamDestroy(w->side);
  if (w->side_gate) cudaEventDestroy(w->side_gate);
  delete w;
}

extern "C" uint64_t tml_struct_size(const char* name) {
  if (!name) return 0;
#define TML_SZ(T) if (!strcmp(name, #T)) return sizeof(T)
  TML_SZ(tml_step_record); TML_SZ(tml_window_row); TML_SZ(tml_proc_record); TML_SZ(tml_live_stats);
  TML_SZ(tml_win_info); TML_SZ(tml_align_info); TML_SZ(tml_reduce_args); TML_SZ(tml_band_args);
  TML_SZ(tml_band_out); TML_SZ(tml_proc_agg); TML_SZ(tml_comm); TML_SZ(tml_reduce_run_args);
  TML_SZ(tml_kind_result); TML_SZ(tml_reduce_run_out); TML_SZ(tml_combined_info); TML_SZ(tml_combined_align);
  TML_SZ(tml_st_diag_in); TML_SZ(tml_mem_diag_in); TML_SZ(tml_proc_diag_in);
  TML_SZ(tml_layer_record);
  TML_SZ(tml_sections_args); TML_SZ(tml_live_phase); TML_SZ(tml_rank_means); TML_SZ(tml_trend_in); TML_SZ(tml_mem_metric_in);
#undef TML_SZ
  return 0;
}
