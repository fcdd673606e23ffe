// Alerts on the GPU: the adds of run_inference (clearcam.py:612-620), the firing loop of process_frame (:465-499) and
// the description alerts of clip_latest_img (:1289-1307), per camera on the tracker handle.  The host form is
// clearcam_b200/alerts.py; this file restates it step for step.  Built with -fmad=false (Makefile): the clock
// comparisons and the similarity sums must round as the host form's do.
//
// State.  Per slot, one device block: every alert's last_det, the object counter (int64 per class), the warm-up count,
// and per (alert, watched class) a ring of `max` timestamps with its head and length.  An alert adds nothing once one of
// its classes holds `max` timestamps, so a ring never overflows.  Alerts without counts (max 0, description alerts) have
// no rings.  The watched classes of an alert are the set bits of its class mask; the ring of class c is the number of set
// bits below c.
//
// Alerts kernel.  One CTA per camera behind a cc_ocsort_gpu_events launch, one warp per alert (alerts are independent).
// The adds of an alert depend on the rows before them (an add can reach `max`), so a warp ballots 32 rows at a time and
// its lane 0 applies them in order.
//
// Describe kernel.  One CTA per camera: a warp per (saved object, description alert) pair sums the products in the
// fixed order of alerts.py `similarity`, then thread 0 walks the saves in order for the cooldown and the first match.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <vector>

#include "cc_common.h"
#include "clearcam_b200.h"
#include "ocsort_gpu.cuh"

using cc::CC_ERR_INVALID;
using cc::CC_OK;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxA = CC_ALERT_MAX_ALERTS;
constexpr int kClasses = CC_OCSORT_CLASSES;
constexpr int kWarmup = 10;                          // process_frame: `if self.count[cam_name] > 10`
constexpr double kDescCooldown = 60.;                // clip_latest_img: `time.time() - v.last_det < 60`

struct AlSlot {
  int A, on, dim, nq;                                // alerts, alerts_on, description width, rings
  char* st;                                          // state block (layout below), nullptr when not configured
  double* last;                                      // [kMaxA]
  long long* counter;                                // [kClasses]
  int* warm;                                         // [1]
  int* qh;                                           // [nq] ring heads
  int* ql;                                           // [nq] ring lengths
  double* ts;                                        // ring timestamps
  float* desc;                                       // [A, dim]
  int qoff[kMaxA];                                   // first ring of each alert
  int toff[kMaxA];                                   // first timestamp of each alert
  cc_alert al[kMaxA];
};

struct Layout {
  size_t last, counter, warm, qh, ql, ts, desc, bytes;
};

Layout layout(int nq, long long nts, int A, int dim) {
  Layout l;
  l.last = 0;
  l.counter = l.last + sizeof(double) * kMaxA;
  l.warm = l.counter + sizeof(long long) * kClasses;
  l.qh = l.warm + 8;
  l.ql = l.qh + sizeof(int) * static_cast<size_t>(nq);
  l.ts = (l.ql + sizeof(int) * static_cast<size_t>(nq) + 7) & ~static_cast<size_t>(7);
  l.desc = l.ts + sizeof(double) * static_cast<size_t>(nts);
  l.bytes = l.desc + sizeof(float) * static_cast<size_t>(A) * dim;
  return l;
}

__host__ __device__ inline int popc3(const uint32_t (&m)[3]) {
#ifdef __CUDA_ARCH__
  return __popc(m[0]) + __popc(m[1]) + __popc(m[2] & 0xffffu);
#else
  return __builtin_popcount(m[0]) + __builtin_popcount(m[1]) + __builtin_popcount(m[2] & 0xffffu);
#endif
}

__device__ inline bool watches(const cc_alert& a, int c) {
  return c >= 0 && c < kClasses && ((a.classes[c >> 5] >> (c & 31)) & 1u);
}
__device__ inline int ring_of(const cc_alert& a, int c) {   // set bits of the mask below class c
  int k = 0;
  for (int w = 0; w < (c >> 5); ++w) k += __popc(a.classes[w]);
  return k + __popc(a.classes[c >> 5] & ((1u << (c & 31)) - 1u));
}
__device__ inline bool keeps_counts(const cc_alert& a) { return a.max > 0 && !(a.flags & CC_ALERT_DESC); }

// RollingClassCounter.is_active (:95-103) at local time (tod seconds of day, wday 0 = Monday)
__device__ bool is_active(const cc_alert& a, int on, double tod, int wday) {
  if (!on || !(a.flags & CC_ALERT_ON)) return false;
  if (!(a.flags & CC_ALERT_SCHED)) return true;
  if (!((a.days >> wday) & 1)) return false;
  return tod < a.end && tod > a.start - a.window;
}

struct AlJob { int slot, wday; double now, tod; };
struct AlJobs { AlJob j[CC_MAX_FRAMES]; };

// One warp: prune every ring of alert `a` at `now` (get_counts); -> whether one holds max timestamps (uniform)
__device__ __forceinline__ bool prune(const AlSlot& s, int a, double now) {
  const cc_alert& al = s.al[a];
  const int nr = popc3(al.classes);
  bool full = false;
  for (int k = threadIdx.x & 31; k < nr; k += 32) {
    const int q = s.qoff[a] + k;
    const double* t = s.ts + s.toff[a] + static_cast<size_t>(k) * al.max;
    int h = s.qh[q], n = s.ql[q];
    while (n > 0 && now - t[h] > al.window) {
      h = h + 1 == al.max ? 0 : h + 1;
      --n;
    }
    s.qh[q] = h;
    s.ql[q] = n;
    full |= n >= al.max;
  }
  return __any_sync(0xffffffffu, full);
}

__global__ void __launch_bounds__(kThreads) alerts_kernel(const __grid_constant__ AlJobs jt, const AlSlot* __restrict__ slots,
                                                          const double* __restrict__ preds, const uint8_t* __restrict__ flags,
                                                          int cap, const int* __restrict__ ev_counts,
                                                          const int* __restrict__ ev_status, int* __restrict__ fired,
                                                          int* __restrict__ res, int B) {
  __shared__ int fire[kMaxA];
  const int b = blockIdx.x;
  if (ev_status[b] != CC_EVENT_OK) {
    if (threadIdx.x == 0) {
      res[b] = 0;
      res[B + b] = CC_ALERT_NOT_RUN;
    }
    return;
  }
  const AlJob job = jt.j[b];
  const AlSlot& s = slots[job.slot];
  const int n = ev_counts[b];
  const double* pr = preds + static_cast<size_t>(b) * cap * 7;
  const uint8_t* fl = flags + static_cast<size_t>(b) * cap;
  const int warm = *s.warm;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;

  for (int i = threadIdx.x; i < n; i += kThreads) {                      // self.counter[cam].add on `new` (:617)
    const int c = static_cast<int>(pr[static_cast<size_t>(i) * 7 + 5]);
    if ((fl[i] & 1) && c >= 0 && c < kClasses) atomicAdd(reinterpret_cast<unsigned long long*>(s.counter + c), 1ull);
  }
  for (int a = threadIdx.x; a < kMaxA; a += kThreads) fire[a] = 0;
  __syncthreads();                                                        // every thread has read the warm-up count
  if (threadIdx.x == 0 && warm <= kWarmup) *s.warm = warm + 1;            // :541, `else: self.count[cam_name] += 1`

  for (int a = w; a < s.A; a += kWarps) {
    const cc_alert& al = s.al[a];
    const bool zone = al.flags & CC_ALERT_ZONE;
    if (keeps_counts(al) && n > 0) {                                      // the adds (:619-620)
      bool full = prune(s, a, job.now);
      __syncwarp();
      for (int c0 = 0; c0 < n && !full; c0 += 32) {
        const int i = c0 + lane;
        bool want = false;
        int c = -1;
        if (i < n) {
          const int f = fl[i];
          c = static_cast<int>(pr[static_cast<size_t>(i) * 7 + 5]);
          want = (((f & 1) && !zone) || ((f & 2) && zone)) && watches(al, c);
        }
        unsigned m = __ballot_sync(0xffffffffu, want);
        if (lane == 0) {
          while (m && !full) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const int cls = static_cast<int>(pr[static_cast<size_t>(c0 + src) * 7 + 5]);
            const int k = ring_of(al, cls);
            const int q = s.qoff[a] + k;
            double* t = s.ts + s.toff[a] + static_cast<size_t>(k) * al.max;
            int h = s.qh[q], len = s.ql[q];
            int tail = h + len;
            if (tail >= al.max) tail -= al.max;
            t[tail] = job.now;
            ++len;
            while (len > 0 && job.now - t[h] > al.window) {              // add's own cleanup
              h = h + 1 == al.max ? 0 : h + 1;
              --len;
            }
            s.qh[q] = h;
            s.ql[q] = len;
            full = len >= al.max;
          }
        }
        full = __shfl_sync(0xffffffffu, full, 0);
        __syncwarp();
      }
    }
    if (warm > kWarmup && !(al.flags & CC_ALERT_DESC)) {                  // the firing loop (:470-499)
      if (!is_active(al, s.on, job.tod, job.wday)) {
        const int nr = keeps_counts(al) ? popc3(al.classes) : 0;
        for (int k = lane; k < nr; k += 32) {
          s.qh[s.qoff[a] + k] = 0;
          s.ql[s.qoff[a] + k] = 0;
        }
      } else if (keeps_counts(al)) {
        const bool full = prune(s, a, job.now);
        if (lane == 0 && full && job.now - s.last[a] >= al.window) {
          s.last[a] = job.now;
          fire[a] = 1;
        }
      }
    }
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int k = 0;
    for (int a = 0; a < s.A; ++a)
      if (fire[a]) fired[static_cast<size_t>(b) * kMaxA + k++] = a;
    res[b] = k;
    res[B + b] = CC_ALERT_OK;
  }
}

struct DsJob { int slot, wday, row0, n; double now, tod; };
struct DsJobs { DsJob j[CC_MAX_FRAMES]; };

__global__ void __launch_bounds__(kThreads) describe_kernel(const __grid_constant__ DsJobs jt, const AlSlot* __restrict__ slots,
                                                            const float* __restrict__ emb, int dim, int* __restrict__ hit,
                                                            float* __restrict__ sim) {
  __shared__ int act[kMaxA];
  const DsJob job = jt.j[blockIdx.x];
  const AlSlot& s = slots[job.slot];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int a = threadIdx.x; a < s.A; a += kThreads)
    act[a] = (s.al[a].flags & CC_ALERT_DESC) && is_active(s.al[a], s.on, job.tod, job.wday);
  const int pairs = job.n * s.A;
  for (int p = w; p < pairs; p += kWarps) {
    const int r = p / s.A, a = p - r * s.A;
    float* out = sim + static_cast<size_t>(job.row0 + r) * kMaxA + a;
    if (!(s.al[a].flags & CC_ALERT_DESC)) {
      if (lane == 0) *out = __int_as_float(0x7fc00000);                  // NaN: no description
      continue;
    }
    const float* e = emb + static_cast<size_t>(job.row0 + r) * dim;
    const float* q = s.desc + static_cast<size_t>(a) * dim;
    double acc = 0.;
    for (int k = lane; k < dim; k += 32) acc += static_cast<double>(e[k]) * static_cast<double>(q[k]);
    for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) *out = static_cast<float>(acc);
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int r = 0; r < job.n; ++r) {
    int h = -1;
    for (int a = 0; a < s.A; ++a) {
      if (job.now - s.last[a] < kDescCooldown || !act[a]) continue;
      const double v = sim[static_cast<size_t>(job.row0 + r) * kMaxA + a];
      if (v > s.al[a].threshold) {
        s.last[a] = job.now;
        h = a;
        break;
      }
    }
    hit[job.row0 + r] = h;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------- host side
struct cc_alerts {
  std::vector<AlSlot> slot;          // host copy of every slot's alerts
  std::vector<std::vector<double>> last;   // per slot: the last_det image pushed by the last configure
  AlSlot* d_slot = nullptr;
};

namespace {

int push_slot(cc_ocsort_gpu* h, int slot, cudaStream_t st) {
  CC_CHECK_CUDA(cudaMemcpyAsync(h->al->d_slot + slot, &h->al->slot[slot], sizeof(AlSlot), cudaMemcpyHostToDevice, st));
  return CC_OK;
}

bool alerts_active(const cc_ocsort_gpu* h, int slot) { return h->al && h->al->slot[slot].st; }

}  // namespace

int cc_alerts_slot_clear(cc_ocsort_gpu* h, int slot, cudaStream_t st) {
  if (!alerts_active(h, slot)) return CC_OK;
  AlSlot& s = h->al->slot[slot];
  CC_CHECK_CUDA(cudaMemsetAsync(s.counter, 0, sizeof(long long) * kClasses + 8, st));   // the counter and the warm-up
  return CC_OK;
}

int cc_alerts_slot_free(cc_ocsort_gpu* h, int slot, cudaStream_t st) {
  if (!alerts_active(h, slot)) return CC_OK;
  CC_CHECK_CUDA(cudaFreeAsync(h->al->slot[slot].st, st));
  h->al->slot[slot] = AlSlot{};
  return push_slot(h, slot, st);
}

void cc_alerts_destroy(cc_ocsort_gpu* h) {
  if (!h->al) return;
  for (auto& s : h->al->slot)
    if (s.st) cudaFree(s.st);
  cudaFree(h->al->d_slot);
  delete h->al;
  h->al = nullptr;
}

extern "C" {

int cc_ocsort_gpu_alerts_configure(cc_ocsort_gpu* h, int slot, const cc_alert* alerts, int n, const float* desc_emb, int dim,
                                   const int* keep, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S, "cc_ocsort_gpu_alerts_configure: bad handle or slot %d", slot);
  CC_REQUIRE(h->cfg[slot].active, "cc_ocsort_gpu_alerts_configure: slot %d is not configured for tracking", slot);
  CC_REQUIRE(n >= 0 && n <= kMaxA, "cc_ocsort_gpu_alerts_configure: %d alerts (0..%d)", n, kMaxA);
  CC_REQUIRE(alerts || n == 0, "cc_ocsort_gpu_alerts_configure: NULL alerts");
  bool any_desc = false;
  for (int i = 0; i < n; ++i) {
    const cc_alert& a = alerts[i];
    CC_REQUIRE(a.max >= 0 && a.max <= CC_ALERT_MAX_COUNT, "cc_ocsort_gpu_alerts_configure: alert %d: max %d (0..%d)", i, a.max,
               CC_ALERT_MAX_COUNT);
    CC_REQUIRE((a.classes[2] >> 16) == 0, "cc_ocsort_gpu_alerts_configure: alert %d: class mask beyond class %d", i, kClasses - 1);
    CC_REQUIRE(isfinite(a.window) && a.window > 0, "cc_ocsort_gpu_alerts_configure: alert %d: window must be finite and > 0", i);
    CC_REQUIRE(isfinite(a.start) && isfinite(a.end) && isfinite(a.last_det) && !isnan(a.threshold),
               "cc_ocsort_gpu_alerts_configure: alert %d: schedule, last_det or threshold not finite", i);
    CC_REQUIRE((a.flags & ~(CC_ALERT_ON | CC_ALERT_ZONE | CC_ALERT_DESC | CC_ALERT_SCHED)) == 0 && (a.days & ~0x7f) == 0,
               "cc_ocsort_gpu_alerts_configure: alert %d: unknown flag or weekday bits", i);
    any_desc |= (a.flags & CC_ALERT_DESC) != 0;
  }
  CC_REQUIRE(!any_desc || (desc_emb && dim >= 1 && dim <= 4096),
             "cc_ocsort_gpu_alerts_configure: description alerts need embeddings of width 1..4096 (got %d)", dim);
  if (!any_desc) dim = 0;
  for (int i = 0; i < n; ++i) {                      // only the rows of description alerts are read
    if (!(alerts[i].flags & CC_ALERT_DESC)) continue;
    for (int k = 0; k < dim; ++k)
      CC_REQUIRE(isfinite(desc_emb[static_cast<size_t>(i) * dim + k]),
                 "cc_ocsort_gpu_alerts_configure: alert %d: description embedding value %d is not finite", i, k);
  }
  const AlSlot* old = h->al ? &h->al->slot[slot] : nullptr;
  for (int i = 0; keep && i < n; ++i) {
    const int k = keep[i];
    if (k < 0) continue;
    CC_REQUIRE(old && old->st && k < old->A, "cc_ocsort_gpu_alerts_configure: alert %d keeps alert %d, which does not exist", i, k);
    const cc_alert &a = alerts[i], &o = old->al[k];
    CC_REQUIRE(a.max == o.max && a.classes[0] == o.classes[0] && a.classes[1] == o.classes[1] && a.classes[2] == o.classes[2] &&
                   (a.flags & CC_ALERT_DESC) == (o.flags & CC_ALERT_DESC),
               "cc_ocsort_gpu_alerts_configure: alert %d keeps alert %d, whose counts differ in shape", i, k);
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!h->al) {
    cc_alerts* e = new cc_alerts();
    e->slot.assign(h->S, AlSlot{});
    e->last.assign(h->S, std::vector<double>());
    cudaError_t r = cudaMalloc(&e->d_slot, sizeof(AlSlot) * h->S);
    if (r == cudaSuccess) r = cudaMemset(e->d_slot, 0, sizeof(AlSlot) * h->S);
    if (r != cudaSuccess) {
      cudaFree(e->d_slot);
      delete e;
      cc::set_error("cc_ocsort_gpu_alerts_configure: %s", cudaGetErrorString(r));
      return cc::CC_ERR_CUDA;
    }
    h->al = e;
    old = &h->al->slot[slot];
  }
  AlSlot ns{};
  ns.A = n;
  ns.on = old->st ? old->on : 1;
  ns.dim = dim;
  long long nts = 0;
  for (int i = 0; i < n; ++i) {
    ns.al[i] = alerts[i];
    ns.qoff[i] = ns.nq;
    ns.toff[i] = static_cast<int>(nts);
    if (alerts[i].max > 0 && !(alerts[i].flags & CC_ALERT_DESC)) {
      const int nr = popc3(alerts[i].classes);
      ns.nq += nr;
      nts += static_cast<long long>(nr) * alerts[i].max;
    }
  }
  const Layout l = layout(ns.nq, nts, n, dim);
  void* p = nullptr;
  CC_CHECK_CUDA(cudaMallocAsync(&p, l.bytes, st));
  ns.st = static_cast<char*>(p);
  ns.last = reinterpret_cast<double*>(ns.st + l.last);
  ns.counter = reinterpret_cast<long long*>(ns.st + l.counter);
  ns.warm = reinterpret_cast<int*>(ns.st + l.warm);
  ns.qh = reinterpret_cast<int*>(ns.st + l.qh);
  ns.ql = reinterpret_cast<int*>(ns.st + l.ql);
  ns.ts = reinterpret_cast<double*>(ns.st + l.ts);
  ns.desc = reinterpret_cast<float*>(ns.st + l.desc);
  std::vector<double>& last = h->al->last[slot];
  last.assign(kMaxA, 0.);
  for (int i = 0; i < n; ++i) last[i] = alerts[i].last_det;
  // every copy into the new block is checked; on a failure the block is freed and the slot keeps its old state
  cudaError_t e = cudaMemsetAsync(ns.st, 0, l.bytes, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(ns.last, last.data(), sizeof(double) * kMaxA, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && dim) e = cudaMemcpyAsync(ns.desc, desc_emb, sizeof(float) * n * dim, cudaMemcpyHostToDevice, st);
  if (old->st) {
    // the object counter and the warm-up stay; kept alerts take their rings and last_det along
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(ns.counter, old->counter, sizeof(long long) * kClasses + 8, cudaMemcpyDeviceToDevice, st);
    for (int i = 0; keep && i < n && e == cudaSuccess; ++i) {
      const int k = keep[i];
      if (k < 0) continue;
      e = cudaMemcpyAsync(ns.last + i, old->last + k, sizeof(double), cudaMemcpyDeviceToDevice, st);
      const int nr = ns.al[i].max > 0 && !(ns.al[i].flags & CC_ALERT_DESC) ? popc3(ns.al[i].classes) : 0;
      if (!nr) continue;
      if (e == cudaSuccess)
        e = cudaMemcpyAsync(ns.qh + ns.qoff[i], old->qh + old->qoff[k], sizeof(int) * nr, cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess)
        e = cudaMemcpyAsync(ns.ql + ns.qoff[i], old->ql + old->qoff[k], sizeof(int) * nr, cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess)
        e = cudaMemcpyAsync(ns.ts + ns.toff[i], old->ts + old->toff[k], sizeof(double) * nr * ns.al[i].max,
                            cudaMemcpyDeviceToDevice, st);
    }
  }
  if (e != cudaSuccess) {
    cudaFreeAsync(p, st);
    cc::set_error("cc_ocsort_gpu_alerts_configure: %s", cudaGetErrorString(e));
    return cc::CC_ERR_CUDA;
  }
  if (old->st) CC_CHECK_CUDA(cudaFreeAsync(old->st, st));
  h->al->slot[slot] = ns;
  return push_slot(h, slot, st);
}

int cc_ocsort_gpu_alerts_set_on(cc_ocsort_gpu* h, int slot, int on, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S && alerts_active(h, slot),
             "cc_ocsort_gpu_alerts_set_on: bad handle, or slot %d has no alerts configured", slot);
  h->al->slot[slot].on = on ? 1 : 0;
  return push_slot(h, slot, static_cast<cudaStream_t>(stream));
}

int cc_ocsort_gpu_alerts_counts(cc_ocsort_gpu* h, int slot, int64_t* counts, void* stream) {
  CC_REQUIRE(h && counts && slot >= 0 && slot < h->S && alerts_active(h, slot),
             "cc_ocsort_gpu_alerts_counts: bad handle or output, or slot %d has no alerts configured", slot);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CC_CHECK_CUDA(cudaMemcpyAsync(counts, h->al->slot[slot].counter, sizeof(int64_t) * kClasses, cudaMemcpyDeviceToHost, st));
  CC_CHECK_CUDA(cudaStreamSynchronize(st));
  return CC_OK;
}

int cc_ocsort_gpu_alerts_reset_counts(cc_ocsort_gpu* h, int slot, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S && alerts_active(h, slot),
             "cc_ocsort_gpu_alerts_reset_counts: bad handle, or slot %d has no alerts configured", slot);
  CC_CHECK_CUDA(cudaMemsetAsync(h->al->slot[slot].counter, 0, sizeof(long long) * kClasses, static_cast<cudaStream_t>(stream)));
  return CC_OK;
}

static int check_local(const char* fn, int b, const double* now, const double* local) {
  CC_REQUIRE(isfinite(now[b]) && isfinite(local[2 * b]), "%s: job %d: the clock or time of day is not finite", fn, b);
  CC_REQUIRE(local[2 * b + 1] >= 0 && local[2 * b + 1] <= 6 && local[2 * b + 1] == floor(local[2 * b + 1]),
             "%s: job %d: weekday %g (0..6)", fn, b, local[2 * b + 1]);
  return CC_OK;
}

int cc_ocsort_gpu_alerts(cc_ocsort_gpu* h, const cc_track_job* jobs, int B, const double* now, const double* local,
                         const double* d_preds, const uint8_t* d_flags, int cap, const int* d_ev_counts, const int* d_ev_status,
                         int* d_fired, int* d_res, void* stream) {
  CC_REQUIRE(h && jobs && now && local && d_preds && d_flags && d_ev_counts && d_ev_status && d_fired && d_res,
             "cc_ocsort_gpu_alerts: NULL argument");
  CC_REQUIRE(B >= 1 && B <= CC_MAX_FRAMES, "cc_ocsort_gpu_alerts: B %d (1..%d)", B, CC_MAX_FRAMES);
  CC_REQUIRE(cap >= 0, "cc_ocsort_gpu_alerts: capacity %d", cap);
  static thread_local std::vector<char> seen;
  seen.assign(h->S, 0);
  AlJobs jt;
  for (int b = 0; b < B; ++b) {
    const int s = jobs[b].slot;
    CC_REQUIRE(s >= 0 && s < h->S && alerts_active(h, s), "cc_ocsort_gpu_alerts: job %d: slot %d has no alerts configured", b, s);
    CC_REQUIRE(!seen[s], "cc_ocsort_gpu_alerts: job %d: slot %d appears twice", b, s);
    const int r = check_local("cc_ocsort_gpu_alerts", b, now, local);
    if (r != CC_OK) return r;
    seen[s] = 1;
    jt.j[b] = AlJob{s, static_cast<int>(local[2 * b + 1]), now[b], local[2 * b]};
  }
  alerts_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(jt, h->al->d_slot, d_preds, d_flags, cap, d_ev_counts,
                                                                        d_ev_status, d_fired, d_res, B);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

int cc_ocsort_gpu_describe(cc_ocsort_gpu* h, const int* slots, const int* rows, int B, const double* now, const double* local,
                           const float* d_emb, int dim, int* d_hit, float* d_sim, void* stream) {
  CC_REQUIRE(h && slots && rows && now && local && d_emb && d_hit && d_sim, "cc_ocsort_gpu_describe: NULL argument");
  CC_REQUIRE(B >= 1 && B <= CC_MAX_FRAMES, "cc_ocsort_gpu_describe: B %d (1..%d)", B, CC_MAX_FRAMES);
  CC_REQUIRE(dim >= 1 && dim <= 4096, "cc_ocsort_gpu_describe: embedding width %d (1..4096)", dim);
  static thread_local std::vector<char> seen;
  seen.assign(h->S, 0);
  DsJobs jt;
  int row0 = 0;
  for (int b = 0; b < B; ++b) {
    const int s = slots[b];
    CC_REQUIRE(s >= 0 && s < h->S && alerts_active(h, s), "cc_ocsort_gpu_describe: job %d: slot %d has no alerts configured", b, s);
    CC_REQUIRE(!seen[s], "cc_ocsort_gpu_describe: job %d: slot %d appears twice", b, s);
    CC_REQUIRE(rows[b] >= 0 && rows[b] <= (1 << 20), "cc_ocsort_gpu_describe: job %d: %d rows", b, rows[b]);
    const AlSlot& al = h->al->slot[s];
    CC_REQUIRE(al.dim == 0 || al.dim == dim, "cc_ocsort_gpu_describe: job %d: embeddings of width %d, descriptions of %d", b, dim,
               al.dim);
    const int r = check_local("cc_ocsort_gpu_describe", b, now, local);
    if (r != CC_OK) return r;
    seen[s] = 1;
    jt.j[b] = DsJob{s, static_cast<int>(local[2 * b + 1]), row0, rows[b], now[b], local[2 * b]};
    row0 += rows[b];
  }
  describe_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(jt, h->al->d_slot, d_emb, dim, d_hit, d_sim);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // extern "C"
