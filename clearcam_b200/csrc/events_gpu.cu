// Object events on the GPU: what run_inference does with the tracker's targets (clearcam.py:586-621), one CTA per
// camera over a cc_ocsort_gpu_update job table, queued right after that launch and reading its outputs.  The host form is
// clearcam_b200/events.py; this file restates it step for step.  Built with -fmad=false (Makefile): the zone test is
// float64 arithmetic that must round as Python's does.
//
// State.  Per slot, one entry per track id that has any (pred_occs / object_set / object_set_zone in the reference): the
// id, flags (bit 0 seen, bit 1 seen in the zone, bits 8.. the occurrence count capped at 20) and the last occurrence
// time.  Entries are kept in ascending id order and only for ids the tracker still holds: a deleted track never comes
// back, so dropping it keeps the reference's unbounded sets exact.  (An id missing from one step's output may be alive
// and return, so absence from the output prunes nothing.)  Each step merges the old entries against the slot's id lane,
// which is strictly ascending (new tracks get increasing ids and compaction keeps order; checked, not assumed), and writes
// the new entries into the other half of a double buffer, so a step that lacks room changes nothing.
//
// Per target.  The tracker's output for one camera holds each live id at most once, in descending id order, so every
// target's decision depends only on its own entry: the targets are decided in parallel and their preds and saves are
// placed by an ordered block compaction, in the reference's order.
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

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxV = CC_EVENT_MAX_VERTICES;
constexpr int kOccCap = 20;                         // clearcam.py:592 `len(...) < 20`
constexpr double kBoxLimit = 1152921504606846976.;  // 2^60: every rectangle step below stays inside int64

enum : int { E_SEEN = 1, E_ZONE = 2, E_OCC_SHIFT = 8 };

struct EvCfg {
  double* last;                      // [2][cap] last occurrence time
  int32_t* id;                       // [2][cap] track id (the tracker's output id)
  int32_t* fl;                       // [2][cap] E_* flags and occurrence count
  int cap, active, nv, outside, nza, filter;
  uint32_t mask[3];
  double zone[2 * kMaxV];
};
struct EvCnt { int n, which; };

struct EvJob { int slot, W, H, pad; double now; };
struct EvJobs { EvJob j[CC_MAX_FRAMES]; };

struct Smem {
  double zx[kMaxV], zy[kMaxV];       // the zone scaled to the frame (clearcam.py:600-601)
  int wc[kWarps];
};

// Exclusive prefix of `flag` in thread order over one chunk of kThreads items; *total (uniform) += the chunk's count.
__device__ int chunk_scan(Smem& sm, bool flag, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  __syncthreads();
  if (lane == 0) sm.wc[w] = __popc(m);
  __syncthreads();
  int off = *total + __popc(m & ((1u << lane) - 1u));
  int sum = 0;
  for (int i = 0; i < kWarps; ++i) {
    if (i < w) off += sm.wc[i];
    sum += sm.wc[i];
  }
  *total += sum;
  return off;
}

// clearcam.py:647-665, in the order and the float64 operations written there
__device__ bool point_not_in_polygon(const double (&c)[4][2], const Smem& sm, int n) {
  for (int j = 0; j < 4; ++j) {
    const double x = c[j][0], y = c[j][1];
    bool inside = false;
    double p1x = sm.zx[0], p1y = sm.zy[0];
    for (int i = 1; i <= n; ++i) {
      const int k = i % n;
      const double p2x = sm.zx[k], p2y = sm.zy[k];
      if (y > fmin(p1y, p2y) && y <= fmax(p1y, p2y) && x <= fmax(p1x, p2x)) {
        const double xi = p1y != p2y ? (y - p1y) * (p2x - p1x) / (p2y - p1y) + p1x : p1x;
        if (p1x == p2x || x <= xi) inside = !inside;
      }
      p1x = p2x;
      p1y = p2y;
    }
    if (inside) return false;
  }
  return true;
}

__device__ inline long long floordiv2(long long a) { return a >= 0 ? a / 2 : -((1 - a) / 2); }   // Python's a // 2
__device__ inline long long clampll(long long v, long long hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

struct View {
  const double* rows;                // this job's tracker rows [n,9]
  int n;
  const EvCfg* cfg;
  int W, H;
  double now;
  __device__ const double* row(int i) const { return rows + static_cast<size_t>(i) * 9; }
  // clearcam.py:586 (class filter) and :589 (tracklet_len)
  __device__ bool considered(int i) const {
    const double* r = row(i);
    const int c = static_cast<int>(r[5]);
    if (cfg->filter && !(c >= 0 && c < 96 && ((cfg->mask[c >> 5] >> (c & 31)) & 1u))) return false;
    return !(r[7] < 1.);
  }
  __device__ bool box_ok(int i) const {
    const double* r = row(i);
    const double v[6] = {r[0], r[1], r[2], r[3], r[0] + r[2], r[1] + r[3]};
    bool ok = true;
    for (int k = 0; k < 6; ++k) ok &= fabs(v[k]) < kBoxLimit;    // false for NaN and infinities too
    return ok;
  }
  // row index of track id `id` (rows are in strictly descending id order), or -1
  __device__ int find_row(int id) const {
    int lo = 0, hi = n;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      const int v = static_cast<int>(row(m)[6]);
      if (v == id) return m;
      if (v > id) lo = m + 1; else hi = m;
    }
    return -1;
  }
};

__device__ int find_id(const int32_t* ids, int n, int id) {   // ascending
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    const int v = ids[m];
    if (v == id) return m;
    if (v < id) lo = m + 1; else hi = m;
  }
  return -1;
}

struct Decision {
  int fl;                            // the entry after this step
  double last;
  bool save, pred;
  uint8_t flags;
  long long rect[4];
};

// One considered target (clearcam.py:591-620) from its entry before this step (fl0 < 0: none).
__device__ Decision decide(const View& v, const Smem& sm, int i, int fl0, double last0) {
  const double* r = v.row(i);
  Decision d;
  d.fl = fl0;
  d.last = last0;
  d.save = d.pred = false;
  d.flags = 0;
  if (fl0 < 0) {                                                  // :591 pred_occs[id] = [time.time()]
    d.fl = 1 << E_OCC_SHIFT;
    d.last = v.now;
  }
  int occ = d.fl >> E_OCC_SHIFT;
  const double dt = v.now - d.last;
  if ((occ < kOccCap && dt > 1.) || dt > 10.) {                   // :592-595, then save_object :380-396
    occ = occ + 1 < kOccCap ? occ + 1 : kOccCap;
    d.fl = (d.fl & 0xff) | (occ << E_OCC_SHIFT);
    d.last = v.now;
    const long long x1 = static_cast<long long>(r[0]), y1 = static_cast<long long>(r[1]);
    const long long x2 = static_cast<long long>(r[0] + r[2]), y2 = static_cast<long long>(r[1] + r[3]);
    const long long cx = floordiv2(x1 + x2), cy = floordiv2(y1 + y2);
    const long long hw = floordiv2(x2 - x1) * 2, hh = floordiv2(y2 - y1) * 2;
    d.rect[0] = clampll(cx - hw, v.W);
    d.rect[2] = clampll(cx + hw, v.W);
    d.rect[1] = clampll(cy - hh, v.H);
    d.rect[3] = clampll(cy + hh, v.H);
    d.save = !(d.rect[3] - d.rect[1] < 100 || d.rect[2] - d.rect[0] < 100);
  }
  if (r[8] < 2.5) return d;                                       // :597
  bool outside = false;
  if (v.cfg->nv > 0) {                                            // :599-603
    const double x1 = r[0], y1 = r[1], x2 = r[0] + r[2], y2 = r[1] + r[3];
    const double c[4][2] = {{x1, y1}, {x2, y1}, {x1, y2}, {x2, y2}};
    outside = point_not_in_polygon(c, sm, v.cfg->nv) != (v.cfg->outside != 0);
  }
  if (outside && !v.cfg->nza) return d;                           // :604-610
  d.pred = true;                                                  // :611-618
  const bool nw = !(d.fl & E_SEEN), nz = !(d.fl & E_ZONE) && !outside;
  d.fl |= (nw ? E_SEEN : 0) | (nz ? E_ZONE : 0);
  d.flags = static_cast<uint8_t>((nw ? 1 : 0) | (nz ? 2 : 0));
  return d;
}

struct EvOut { int status, n_preds, n_saves; };

// One step of slot job.slot's events (the whole CTA) on one frame's tracker rows trk [n,9], with the tracker's live ids
// lane [T] (ascending) after that frame; outputs into po [cap,7], fo [cap], so [cap,6].  Returns (uniform) the status and
// the row counts (for NEEDS_ROOM, n_preds = the capacity needed).
__device__ __forceinline__ EvOut events_frame(Smem& sm, const EvJob job, const EvCfg* ecfgs, EvCnt* ecnts,
                                              const double* __restrict__ trk, int n, const int32_t* __restrict__ lane, int T,
                                              double* __restrict__ po, uint8_t* __restrict__ fo, long long* __restrict__ so) {
  auto finish = [&](int st, int n_preds, int n_saves) { return EvOut{st, n_preds, n_saves}; };
  const EvCfg* cfg = ecfgs + job.slot;
  const View v{trk, n, cfg, job.W, job.H, job.now};
  const int nv = cfg->nv;
  for (int k = threadIdx.x; k < nv; k += kThreads) {
    sm.zx[k] = cfg->zone[2 * k] * static_cast<double>(job.W);
    sm.zy[k] = cfg->zone[2 * k + 1] * static_cast<double>(job.H);
  }

  // ---- checks before anything changes
  bool bad_box = false, bad_order = false;
  for (int t = threadIdx.x + 1; t < T; t += kThreads) bad_order |= lane[t - 1] >= lane[t];
  for (int i = threadIdx.x; i < v.n; i += kThreads) {
    if (i > 0) bad_order |= !(v.row(i - 1)[6] > v.row(i)[6]);
    bad_box |= v.considered(i) && !v.box_ok(i);
  }
  if (__syncthreads_or(bad_box)) return finish(CC_EVENT_BAD_BOX, 0, 0);
  if (__syncthreads_or(bad_order)) return finish(CC_EVENT_BAD_ORDER, 0, 0);

  const EvCnt ec = ecnts[job.slot];
  const size_t o_old = static_cast<size_t>(ec.which) * cfg->cap, o_new = static_cast<size_t>(1 - ec.which) * cfg->cap;
  const int32_t* old_id = cfg->id + o_old;
  const int32_t* old_fl = cfg->fl + o_old;
  const double* old_last = cfg->last + o_old;

  // ---- the entries after this step: a live id keeps its entry, a considered target without one gets one
  auto has = [&](int t, int* jo, int* jr) {
    const int id = lane[t] + 1;                                   // the output's track_id
    *jo = find_id(old_id, ec.n, id);
    *jr = v.find_row(id);
    if (*jr >= 0 && !v.considered(*jr)) *jr = -1;
    return *jo >= 0 || *jr >= 0;
  };
  int need = 0;
  for (int c0 = 0; c0 < T; c0 += kThreads) {
    const int t = c0 + threadIdx.x;
    int jo, jr;
    need += __syncthreads_count(t < T && has(t, &jo, &jr));
  }
  if (need > cfg->cap) return finish(CC_EVENT_NEEDS_ROOM, need, 0);

  int pos = 0;
  for (int c0 = 0; c0 < T; c0 += kThreads) {
    const int t = c0 + threadIdx.x;
    int jo = -1, jr = -1;
    const bool h = t < T && has(t, &jo, &jr);
    const int p = chunk_scan(sm, h, &pos);
    if (!h) continue;
    int fl = jo >= 0 ? old_fl[jo] : -1;
    double last = jo >= 0 ? old_last[jo] : 0.;
    if (jr >= 0) {
      const Decision d = decide(v, sm, jr, fl, last);
      fl = d.fl;
      last = d.last;
    }
    cfg->id[o_new + p] = lane[t] + 1;
    cfg->fl[o_new + p] = fl;
    cfg->last[o_new + p] = last;
  }

  // ---- outputs in target order: preds rows with their flags, and the saves
  int np_ = 0, ns_ = 0;
  for (int c0 = 0; c0 < v.n; c0 += kThreads) {
    const int i = c0 + threadIdx.x;
    Decision d;
    d.save = d.pred = false;
    if (i < v.n && v.considered(i)) {
      const int jo = find_id(old_id, ec.n, static_cast<int>(v.row(i)[6]));
      d = decide(v, sm, i, jo >= 0 ? old_fl[jo] : -1, jo >= 0 ? old_last[jo] : 0.);
    }
    const int pp = chunk_scan(sm, d.pred, &np_);
    const int sp = chunk_scan(sm, d.save, &ns_);
    const double* r = i < v.n ? v.row(i) : nullptr;
    if (d.pred) {
      double* o = po + static_cast<size_t>(pp) * 7;
      o[0] = r[0];
      o[1] = r[1];
      o[2] = r[0] + r[2];
      o[3] = r[1] + r[3];
      o[4] = r[4];
      o[5] = r[5];
      o[6] = r[6];
      fo[pp] = d.flags;
    }
    if (d.save) {
      long long* o = so + static_cast<size_t>(sp) * 6;
      o[0] = static_cast<long long>(r[6]);
      o[1] = static_cast<long long>(r[5]);
      for (int k = 0; k < 4; ++k) o[2 + k] = d.rect[k];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) ecnts[job.slot] = EvCnt{need, 1 - ec.which};
  return finish(CC_EVENT_OK, np_, ns_);
}

__global__ void __launch_bounds__(kThreads) events_kernel(const __grid_constant__ EvJobs jt, const ocsg::SlotCfg* __restrict__ tcfg,
                                                          const ocsg::SlotCnt* __restrict__ tcnt, const EvCfg* __restrict__ ecfgs,
                                                          EvCnt* __restrict__ ecnts, const double* __restrict__ trk_out, int trk_cap,
                                                          const int* __restrict__ trk_count, const int* __restrict__ trk_status,
                                                          double* __restrict__ preds, uint8_t* __restrict__ flags,
                                                          long long* __restrict__ saves, int cap, int* __restrict__ counts,
                                                          int* __restrict__ status, int B) {
  __shared__ Smem sm;
  const int b = blockIdx.x;
  const EvJob job = jt.j[b];
  auto finish = [&](const EvOut& r) {
    if (threadIdx.x == 0) {
      counts[b] = r.n_preds;
      counts[B + b] = r.n_saves;
      status[b] = r.status;
    }
  };
  if (trk_status[b] != CC_TRACK_OK) return finish(EvOut{CC_EVENT_NOT_RUN, 0, 0});
  const ocsg::SlotCfg tc = tcfg[job.slot];
  finish(events_frame(sm, job, ecfgs, ecnts, trk_out + static_cast<size_t>(b) * trk_cap * 9, trk_count[b],
                      tc.il + static_cast<size_t>(ocsg::kLaneId) * tc.cap, tcnt[job.slot].T, preds + static_cast<size_t>(b) * cap * 7,
                      flags + static_cast<size_t>(b) * cap, saves + static_cast<size_t>(b) * cap * 6));
}

// Runs (cc_ocsort_gpu_events_runs): job b's CTA applies the frames its tracker run completed, in order, each on that
// frame's tracker rows and live ids, and stops at the first frame whose status is not OK.  Per-frame picture sizes and
// clocks travel in the parameter block; a call with more frames is split into launches of at most kRunFrames.
constexpr int kRunFrames = 1024;
struct EvRun { int slot, frames, f0, pad; };
struct EvFrame { int W, H; double now; };
struct EvRuns {
  EvRun r[CC_MAX_FRAMES];
  EvFrame f[kRunFrames];
  int b0;                              // first job of this launch
};

// The slot's entries are read back frame after frame: no __restrict__ on `ecfgs` / `ecnts`, so none of them is loaded
// through the read-only (non-coherent) path.
__global__ void __launch_bounds__(kThreads) events_run_kernel(const __grid_constant__ EvRuns rt, const EvCfg* ecfgs,
                                                              EvCnt* ecnts, int tmax, const double* __restrict__ trk_out,
                                                              int trk_cap, const int* __restrict__ trk_count,
                                                              const int32_t* __restrict__ trk_ids, int id_cap,
                                                              const int* __restrict__ trk_live, const int* __restrict__ trk_done,
                                                              double* __restrict__ preds, uint8_t* __restrict__ flags,
                                                              long long* __restrict__ saves, int cap, int* __restrict__ counts,
                                                              int* __restrict__ done, int* __restrict__ status, int B) {
  __shared__ Smem sm;
  const EvRun run = rt.r[blockIdx.x];
  const int b = rt.b0 + blockIdx.x;
  const int frames = min(run.frames, trk_done[b]);
  int f = 0, st = CC_EVENT_OK;
  for (; f < frames; ++f) {
    const size_t bf = static_cast<size_t>(b) * tmax + f;
    const EvFrame fr = rt.f[run.f0 + f];
    const EvOut r = events_frame(sm, EvJob{run.slot, fr.W, fr.H, 0, fr.now}, ecfgs, ecnts, trk_out + bf * trk_cap * 9, trk_count[bf],
                                 trk_ids + bf * id_cap, trk_live[bf], preds + bf * cap * 7, flags + bf * cap, saves + bf * cap * 6);
    if (threadIdx.x == 0) {
      counts[bf] = r.n_preds;
      counts[static_cast<size_t>(B) * tmax + bf] = r.n_saves;
    }
    if (r.status != CC_EVENT_OK) {
      st = r.status;
      break;
    }
    __syncthreads();                   // the slot's entries as this frame left them, for the next
  }
  if (threadIdx.x == 0) {
    done[b] = f;
    status[b] = st == CC_EVENT_OK && f < run.frames ? CC_EVENT_NOT_RUN : st;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------- host side
struct cc_events {
  std::vector<EvCfg> cfg;            // host copy of every slot's event configuration
  EvCfg* d_cfg = nullptr;
  EvCnt* d_cnt = nullptr;
};

namespace {

constexpr size_t kEntryBytes = 2 * (sizeof(double) + 2 * sizeof(int32_t));   // both halves of the double buffer

int alloc_events(int cap, cudaStream_t st, EvCfg& c) {
  void* p = nullptr;
  CC_CHECK_CUDA(cudaMallocAsync(&p, static_cast<size_t>(cap) * kEntryBytes, st));
  c.last = static_cast<double*>(p);
  c.id = reinterpret_cast<int32_t*>(c.last + 2 * static_cast<size_t>(cap));
  c.fl = c.id + 2 * static_cast<size_t>(cap);
  c.cap = cap;
  return CC_OK;
}

int push_events(cc_ocsort_gpu* h, int slot, cudaStream_t st) {
  CC_CHECK_CUDA(cudaMemcpyAsync(h->ev->d_cfg + slot, &h->ev->cfg[slot], sizeof(EvCfg), cudaMemcpyHostToDevice, st));
  return CC_OK;
}

bool events_active(const cc_ocsort_gpu* h, int slot) { return h->ev && h->ev->cfg[slot].active; }

}  // namespace

int cc_events_slot_clear(cc_ocsort_gpu* h, int slot, cudaStream_t st) {
  if (!events_active(h, slot)) return CC_OK;
  CC_CHECK_CUDA(cudaMemsetAsync(h->ev->d_cnt + slot, 0, sizeof(EvCnt), st));
  return CC_OK;
}

int cc_events_slot_free(cc_ocsort_gpu* h, int slot, cudaStream_t st) {
  if (!events_active(h, slot)) return CC_OK;
  EvCfg& c = h->ev->cfg[slot];
  CC_CHECK_CUDA(cudaFreeAsync(c.last, st));
  c = EvCfg{};
  return push_events(h, slot, st);
}

void cc_events_destroy(cc_ocsort_gpu* h) {
  if (!h->ev) return;
  for (auto& c : h->ev->cfg)
    if (c.active) cudaFree(c.last);
  cudaFree(h->ev->d_cfg);
  cudaFree(h->ev->d_cnt);
  delete h->ev;
  h->ev = nullptr;
}

extern "C" {

int cc_ocsort_gpu_events_configure(cc_ocsort_gpu* h, int slot, const double* zone_xy, int n_vertices, int outside,
                                   int non_zone_alert, const uint32_t* class_mask, int capacity, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S, "cc_ocsort_gpu_events_configure: bad handle or slot %d", slot);
  CC_REQUIRE(h->cfg[slot].active, "cc_ocsort_gpu_events_configure: slot %d is not configured for tracking", slot);
  CC_REQUIRE(n_vertices >= 0 && n_vertices <= kMaxV, "cc_ocsort_gpu_events_configure: %d zone vertices (0..%d)", n_vertices, kMaxV);
  CC_REQUIRE(zone_xy || n_vertices == 0, "cc_ocsort_gpu_events_configure: NULL zone with %d vertices", n_vertices);
  for (int k = 0; k < 2 * n_vertices; ++k)
    CC_REQUIRE(isfinite(zone_xy[k]), "cc_ocsort_gpu_events_configure: zone coordinate %d is not finite", k);
  CC_REQUIRE(capacity >= 1 && capacity <= (1 << 20), "cc_ocsort_gpu_events_configure: capacity %d (1..%d)", capacity, 1 << 20);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!h->ev) {
    cc_events* e = new cc_events();
    e->cfg.assign(h->S, EvCfg{});
    cudaError_t r = cudaMalloc(&e->d_cfg, sizeof(EvCfg) * h->S);
    if (r == cudaSuccess) r = cudaMalloc(&e->d_cnt, sizeof(EvCnt) * h->S);
    if (r == cudaSuccess) r = cudaMemset(e->d_cfg, 0, sizeof(EvCfg) * h->S);
    if (r == cudaSuccess) r = cudaMemset(e->d_cnt, 0, sizeof(EvCnt) * h->S);
    if (r != cudaSuccess) {
      cudaFree(e->d_cfg);
      cudaFree(e->d_cnt);
      delete e;
      cc::set_error("cc_ocsort_gpu_events_configure: %s", cudaGetErrorString(r));
      return cc::CC_ERR_CUDA;
    }
    h->ev = e;
  }
  EvCfg& c = h->ev->cfg[slot];
  if (c.active && c.cap != capacity) {
    CC_CHECK_CUDA(cudaFreeAsync(c.last, st));
    c.active = 0;
  }
  if (!c.active) {
    const int r = alloc_events(capacity, st, c);
    if (r != CC_OK) return r;
  }
  c.active = 1;
  c.nv = n_vertices;
  c.outside = outside ? 1 : 0;
  c.nza = non_zone_alert ? 1 : 0;
  c.filter = class_mask != nullptr;
  for (int k = 0; k < 3; ++k) c.mask[k] = class_mask ? class_mask[k] : 0xffffffffu;
  for (int k = 0; k < 2 * kMaxV; ++k) c.zone[k] = k < 2 * n_vertices ? zone_xy[k] : 0.;
  CC_CHECK_CUDA(cudaMemsetAsync(h->ev->d_cnt + slot, 0, sizeof(EvCnt), st));
  return push_events(h, slot, st);
}

int cc_ocsort_gpu_events_grow(cc_ocsort_gpu* h, int slot, int capacity, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S, "cc_ocsort_gpu_events_grow: bad handle or slot %d", slot);
  CC_REQUIRE(events_active(h, slot), "cc_ocsort_gpu_events_grow: slot %d is not configured for events", slot);
  CC_REQUIRE(capacity <= (1 << 20), "cc_ocsort_gpu_events_grow: capacity %d too large", capacity);
  EvCfg& c = h->ev->cfg[slot];
  if (capacity <= c.cap) return CC_OK;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  EvCfg n = c;
  const int r = alloc_events(capacity, st, n);
  if (r != CC_OK) return r;
  // both halves of every region keep their first c.cap entries: one strided copy per region
  CC_CHECK_CUDA(cudaMemcpy2DAsync(n.last, n.cap * sizeof(double), c.last, c.cap * sizeof(double), c.cap * sizeof(double), 2,
                                  cudaMemcpyDeviceToDevice, st));
  CC_CHECK_CUDA(cudaMemcpy2DAsync(n.id, n.cap * 4, c.id, c.cap * 4, c.cap * 4, 2, cudaMemcpyDeviceToDevice, st));
  CC_CHECK_CUDA(cudaMemcpy2DAsync(n.fl, n.cap * 4, c.fl, c.cap * 4, c.cap * 4, 2, cudaMemcpyDeviceToDevice, st));
  CC_CHECK_CUDA(cudaFreeAsync(c.last, st));
  c = n;
  return push_events(h, slot, st);
}

int cc_ocsort_gpu_events_set_non_zone_alert(cc_ocsort_gpu* h, int slot, int non_zone_alert, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S, "cc_ocsort_gpu_events_set_non_zone_alert: bad handle or slot %d", slot);
  CC_REQUIRE(events_active(h, slot), "cc_ocsort_gpu_events_set_non_zone_alert: slot %d is not configured for events", slot);
  h->ev->cfg[slot].nza = non_zone_alert ? 1 : 0;
  return push_events(h, slot, static_cast<cudaStream_t>(stream));
}

int cc_ocsort_gpu_events(cc_ocsort_gpu* h, const cc_track_job* jobs, int B, const int* frame_wh, const double* now,
                         const double* d_trk_out, int trk_cap, const int* d_trk_count, const int* d_trk_status, double* d_preds,
                         uint8_t* d_flags, int64_t* d_saves, int cap, int* d_counts, int* d_status, void* stream) {
  CC_REQUIRE(h && jobs && frame_wh && now && d_trk_out && d_trk_count && d_trk_status && d_preds && d_flags && d_saves &&
                 d_counts && d_status,
             "cc_ocsort_gpu_events: NULL argument");
  CC_REQUIRE(B >= 1 && B <= CC_MAX_FRAMES, "cc_ocsort_gpu_events: B %d (1..%d)", B, CC_MAX_FRAMES);
  CC_REQUIRE(trk_cap >= 0 && cap >= trk_cap, "cc_ocsort_gpu_events: output capacity %d below the tracker's %d", cap, trk_cap);
  static thread_local std::vector<char> seen;
  seen.assign(h->S, 0);
  EvJobs jt;
  for (int b = 0; b < B; ++b) {
    const int s = jobs[b].slot;
    CC_REQUIRE(s >= 0 && s < h->S && h->cfg[s].active && events_active(h, s),
               "cc_ocsort_gpu_events: job %d: slot %d is not configured for tracking and events", b, s);
    CC_REQUIRE(!seen[s], "cc_ocsort_gpu_events: job %d: slot %d appears twice", b, s);
    CC_REQUIRE(frame_wh[2 * b] >= 1 && frame_wh[2 * b + 1] >= 1, "cc_ocsort_gpu_events: job %d: frame %d x %d", b,
               frame_wh[2 * b], frame_wh[2 * b + 1]);
    CC_REQUIRE(isfinite(now[b]), "cc_ocsort_gpu_events: job %d: the clock is not finite", b);
    seen[s] = 1;
    jt.j[b] = EvJob{s, frame_wh[2 * b], frame_wh[2 * b + 1], 0, now[b]};
  }
  events_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      jt, h->d_cfg, h->d_cnt, h->ev->d_cfg, h->ev->d_cnt, d_trk_out, trk_cap, d_trk_count, d_trk_status, d_preds, d_flags,
      reinterpret_cast<long long*>(d_saves), cap, d_counts, d_status, B);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

int cc_ocsort_gpu_events_runs(cc_ocsort_gpu* h, const cc_track_run* runs, int B, int frames_max, const int* frame_wh, const double* now,
                              const double* d_trk_out, int trk_cap, const int* d_trk_count, const int32_t* d_trk_ids, int id_cap,
                              const int* d_trk_live, const int* d_trk_done, double* d_preds, uint8_t* d_flags, int64_t* d_saves, int cap,
                              int* d_counts, int* d_done, int* d_status, void* stream) {
  CC_REQUIRE(h && runs && frame_wh && now && d_trk_out && d_trk_count && d_trk_ids && d_trk_live && d_trk_done && d_preds && d_flags &&
                 d_saves && d_counts && d_done && d_status,
             "cc_ocsort_gpu_events_runs: NULL argument");
  CC_REQUIRE(B >= 1 && B <= CC_MAX_FRAMES && frames_max >= 1 && frames_max <= CC_MAX_FRAMES,
             "cc_ocsort_gpu_events_runs: B %d, frames_max %d (1..%d)", B, frames_max, CC_MAX_FRAMES);
  CC_REQUIRE(trk_cap >= 0 && cap >= trk_cap && id_cap >= 1, "cc_ocsort_gpu_events_runs: output capacity %d below the tracker's %d",
             cap, trk_cap);
  static thread_local std::vector<char> seen;
  seen.assign(h->S, 0);
  int f0 = 0;
  for (int b = 0; b < B; ++b) {
    const int s = runs[b].slot, T = runs[b].frames;
    CC_REQUIRE(s >= 0 && s < h->S && h->cfg[s].active && events_active(h, s),
               "cc_ocsort_gpu_events_runs: run %d: slot %d is not configured for tracking and events", b, s);
    CC_REQUIRE(!seen[s], "cc_ocsort_gpu_events_runs: run %d: slot %d appears twice", b, s);
    CC_REQUIRE(T >= 1 && T <= frames_max, "cc_ocsort_gpu_events_runs: run %d: %d frames (1..%d)", b, T, frames_max);
    for (int f = f0; f < f0 + T; ++f) {
      CC_REQUIRE(frame_wh[2 * f] >= 1 && frame_wh[2 * f + 1] >= 1, "cc_ocsort_gpu_events_runs: run %d frame %d: %d x %d", b, f - f0,
                 frame_wh[2 * f], frame_wh[2 * f + 1]);
      CC_REQUIRE(isfinite(now[f]), "cc_ocsort_gpu_events_runs: run %d frame %d: the clock is not finite", b, f - f0);
    }
    seen[s] = 1;
    f0 += T;
  }
  // launches of consecutive runs with at most kRunFrames frames in all
  static thread_local EvRuns rt;
  for (int b = 0, f = 0; b < B;) {
    int nb = 0, nf = 0;
    rt.b0 = b;
    while (b + nb < B && nf + runs[b + nb].frames <= kRunFrames) {
      const cc_track_run& r = runs[b + nb];
      rt.r[nb] = EvRun{r.slot, r.frames, nf, 0};
      for (int k = 0; k < r.frames; ++k, ++f) rt.f[nf + k] = EvFrame{frame_wh[2 * f], frame_wh[2 * f + 1], now[f]};
      nf += r.frames;
      ++nb;
    }
    events_run_kernel<<<nb, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        rt, h->ev->d_cfg, h->ev->d_cnt, frames_max, d_trk_out, trk_cap, d_trk_count, d_trk_ids, id_cap, d_trk_live, d_trk_done, d_preds,
        d_flags, reinterpret_cast<long long*>(d_saves), cap, d_counts, d_done, d_status, B);
    CC_CHECK_CUDA(cudaGetLastError());
    b += nb;
  }
  return CC_OK;
}

}  // extern "C"
