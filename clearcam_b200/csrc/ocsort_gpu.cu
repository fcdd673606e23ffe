// Device OC-SORT: the trackers of many cameras stepped in ONE launch, one CTA per camera, bit for bit the host tracker of
// ocsort.cu (track ids included).  The per-track arithmetic is ocsort_math.cuh, shared with the host; this file restates
// only the control flow of cc_ocsort::update, stage by stage and in its order.  Built with -fmad=false (Makefile).
//
// State.  A handle owns S camera slots.  Per slot, host-written configuration (SlotCfg: storage, capacity, OCSort
// arguments) and device-written counters (SlotCnt: live tracks T, frame count, next id).  A slot's tracks live in
// structure-of-arrays form with the slot's capacity as stride: `dl` holds ND lanes of doubles, `il` NI lanes of 4-byte
// ints / floats, element t of lane L at L * cap + t.  Class votes are a dense float[80] per track plus the insertion
// order of the classes seen (80 bytes), so `best` is the FIRST maximum in insertion order as in the host's vector.
//
// Capacity.  A frame adds at most D tracks (D = detections above the threshold), so a CTA first checks T + D <= cap; if
// not it changes nothing, reports CC_TRACK_NEEDS_ROOM with the count it needs, and the host grows the slot
// (cc_ocsort_gpu_grow: one strided copy per region) and relaunches that camera.
//
// Assignment.  The host walks all pairs in (cost, flat index) order and takes a pair when its row and column are free.
// Here each free row keeps its minimum over the free columns (first minimum = smallest flat index); every round takes the
// smallest (minimum, flat index) over the rows, then rescans only the rows whose minimum sat in the column just taken.
// That accepts exactly the host's pairs in the host's order.  Costs are recomputed from the boxes when needed rather
// than stored, so no D x T matrix is ever held.
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "cc_common.h"
#include "clearcam_b200.h"
#include "ocsort_gpu.cuh"
#include "ocsort_math.cuh"

using cc::CC_ERR_INVALID;
using cc::CC_OK;

namespace {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kClasses = CC_OCSORT_CLASSES;

// ---- double lanes
enum : int {
  D_X = 0, D_P = 7, D_SX = 56, D_SP = 63, D_HM = 112, D_SHM = 120, D_VEL = 128, D_AVG = 130, D_SPEED = 132,
  D_KEEP = 133,                      // lanes below move with a track when the slot is compacted
  D_TRK = 133, D_LASTB = 137,        // per-frame: predicted box, last observation before this frame's updates,
  D_ANC = 141,                       // and the angle cost's anchor (valid, cx, cy of the observation delta_t back)
  ND = 144
};
// ---- 4-byte lanes; the observation ring (age + box per entry, oldest first) and the scratch lanes follow I_OBS
enum : int {
  I_HLEN = 0, I_HIDX = 1, I_HFL = 3, I_SHLEN = 5, I_SHIDX = 6, I_SHFL = 8, I_KFL = 10, I_ID = 11, I_AGE = 12, I_HITS = 13,
  I_STREAK = 14, I_TSU = 15, I_HASLAST = 16, I_LAST = 17, I_SCORE = 22, I_CLASS = 23, I_NOCC = 24, I_OCC = 25,
  I_OCCL = I_OCC + kClasses, I_NOBS = I_OCCL + kClasses / 4, I_OBS = I_NOBS + 1
};
__host__ __device__ inline int lane_keep(int rb) { return I_OBS + 6 * rb; }   // 4-byte lanes that move with a track
__host__ __device__ inline int lane_count(int rb) { return lane_keep(rb) + 4; }
// scratch lanes (relative to lane_keep): column used (assignment), un_trks list, per-track flags, output slot
enum : int { S_COLUSED = 0, S_UTRK = 1, S_FLAGS = 2, S_POS = 3 };
enum : int { F_MATCHED = 1, F_INUT = 2, F_REMOVED = 4 };

using ocsg::SlotCfg;
using ocsg::SlotCnt;
static_assert(I_ID == ocsg::kLaneId, "events_gpu.cu reads the id lane");

struct JobTable { cc_track_job j[CC_MAX_FRAMES]; };

struct Tr {
  double* dl;
  int32_t* il;
  int cap, scr;
  __device__ double& d(int lane, int t) const { return dl[static_cast<size_t>(lane) * cap + t]; }
  __device__ int32_t& i(int lane, int t) const { return il[static_cast<size_t>(lane) * cap + t]; }
  __device__ float& f(int lane, int t) const { return reinterpret_cast<float*>(il)[static_cast<size_t>(lane) * cap + t]; }
  __device__ int32_t& s(int k, int t) const { return i(scr + k, t); }
};

// ------------------------------------------------------------------------------------------------- track state <-> Kalman
// Loops kept rolled: the Kalman state lives in the thread's stack frame rather than in (spilled) registers.
__device__ void load_hist(const Tr& s, int t, int il, int dl, ocs::History& h) {
  h.len = s.i(il, t);
  h.idx[0] = s.i(il + 1, t);
  h.idx[1] = s.i(il + 2, t);
#pragma unroll 1
  for (int m = 0; m < 2; ++m) {
    const int fl = s.i(il + 3 + m, t);
    h.m[m].some = fl & 1;
    h.m[m].f32 = (fl >> 1) & 1;
    for (int k = 0; k < 4; ++k) h.m[m].v[k] = s.d(dl + m * 4 + k, t);
  }
}
__device__ void store_hist(const Tr& s, int t, int il, int dl, const ocs::History& h) {
  s.i(il, t) = h.len;
  s.i(il + 1, t) = h.idx[0];
  s.i(il + 2, t) = h.idx[1];
#pragma unroll 1
  for (int m = 0; m < 2; ++m) {
    s.i(il + 3 + m, t) = (h.m[m].some ? 1 : 0) | (h.m[m].f32 ? 2 : 0);
    for (int k = 0; k < 4; ++k) s.d(dl + m * 4 + k, t) = h.m[m].v[k];
  }
}
__device__ void load_kf(const Tr& s, int t, ocs::Kalman& k) {
#pragma unroll 1
  for (int i = 0; i < 7; ++i) k.x[i] = s.d(D_X + i, t);
#pragma unroll 1
  for (int i = 0; i < 49; ++i) k.P[i] = s.d(D_P + i, t);
#pragma unroll 1
  for (int i = 0; i < 7; ++i) k.sx[i] = s.d(D_SX + i, t);
#pragma unroll 1
  for (int i = 0; i < 49; ++i) k.sP[i] = s.d(D_SP + i, t);
  load_hist(s, t, I_HLEN, D_HM, k.hist);
  load_hist(s, t, I_SHLEN, D_SHM, k.shist);
  const int fl = s.i(I_KFL, t);
  k.observed = fl & 1;
  k.has_saved = (fl >> 1) & 1;
}
__device__ void store_kf(const Tr& s, int t, const ocs::Kalman& k) {
#pragma unroll 1
  for (int i = 0; i < 7; ++i) s.d(D_X + i, t) = k.x[i];
#pragma unroll 1
  for (int i = 0; i < 49; ++i) s.d(D_P + i, t) = k.P[i];
#pragma unroll 1
  for (int i = 0; i < 7; ++i) s.d(D_SX + i, t) = k.sx[i];
#pragma unroll 1
  for (int i = 0; i < 49; ++i) s.d(D_SP + i, t) = k.sP[i];
  store_hist(s, t, I_HLEN, D_HM, k.hist);
  store_hist(s, t, I_SHLEN, D_SHM, k.shist);
  s.i(I_KFL, t) = (k.observed ? 1 : 0) | (k.has_saved ? 2 : 0);
}

__device__ __noinline__ void track_none(const Tr& s, int t) {   // kalmanfilter.py:109-117
  ocs::Kalman kf;
  load_kf(s, t, kf);
  kf.update_none();
  store_kf(s, t, kf);
}

__device__ bool last_nonneg(const Tr& s, int t) {
  if (!s.i(I_HASLAST, t)) return false;
  float b[5];
  for (int k = 0; k < 5; ++k) b[k] = s.f(I_LAST + k, t);
  return ocs::box_sum_nonneg(b);
}

// The observation delta_t frames back (ocsort.py:11-19): the ring entry of age age - (delta_t - i) for the first i = 0..
// that has one, else -1 (the callers fall back to the last observation or the newest entry, as the host does).
__device__ int find_obs(const Tr& s, int t, int age, int delta_t) {
  const int n = s.i(I_NOBS, t);
  for (int i = 0; i < delta_t; ++i)
    for (int k = n - 1; k >= 0; --k)
      if (s.i(I_OBS + 6 * k, t) == age - (delta_t - i)) return k;
  return -1;
}

// ocsort.py:105-139 with a detection (row r = x1,y1,x2,y2,score,class)
// Out of line, like every function below that holds a Kalman state: each keeps its own frame instead of spilling.
__device__ __noinline__ void track_update(const Tr& s, int t, const float* r, int delta_t) {
  const int cls = static_cast<int>(r[5]);
  const float score = r[4];
  const int nocc = s.i(I_NOCC, t);
  bool seen = false;
  for (int k = 0; k < nocc && !seen; ++k) seen = ((s.i(I_OCCL + k / 4, t) >> (8 * (k % 4))) & 0xff) == cls;
  if (seen) {
    s.f(I_OCC + cls, t) += score;
  } else {
    s.f(I_OCC + cls, t) = score;
    int32_t& w = s.i(I_OCCL + nocc / 4, t);
    const int sh = 8 * (nocc % 4);
    w = static_cast<int32_t>((static_cast<uint32_t>(w) & ~(0xffu << sh)) | (static_cast<uint32_t>(cls) << sh));
    s.i(I_NOCC, t) = nocc + 1;
  }
  {
    const int n = seen ? nocc : nocc + 1;
    int c0 = s.i(I_OCCL, t) & 0xff;
    float best = s.f(I_OCC + c0, t);
    int best_c = c0;
    for (int k = 1; k < n; ++k) {
      const int c = (s.i(I_OCCL + k / 4, t) >> (8 * (k % 4))) & 0xff;
      const float v = s.f(I_OCC + c, t);
      if (v > best) { best = v; best_c = c; }
    }
    s.i(I_CLASS, t) = best_c;
  }
  const int age = s.i(I_AGE, t);
  if (last_nonneg(s, t)) {
    float prev[5];
    const int k = find_obs(s, t, age, delta_t);
    for (int j = 0; j < 5; ++j) prev[j] = k >= 0 ? s.f(I_OBS + 6 * k + 1 + j, t) : s.f(I_LAST + j, t);
    double vel[2] = {s.d(D_VEL, t), s.d(D_VEL + 1, t)}, avg[2] = {s.d(D_AVG, t), s.d(D_AVG + 1, t)}, speed;
    ocs::velocity_update(prev, r, age, vel, avg, &speed);
    s.d(D_VEL, t) = vel[0];
    s.d(D_VEL + 1, t) = vel[1];
    s.d(D_AVG, t) = avg[0];
    s.d(D_AVG + 1, t) = avg[1];
    s.d(D_SPEED, t) = speed;
  }
  for (int j = 0; j < 5; ++j) s.f(I_LAST + j, t) = r[j];
  s.i(I_HASLAST, t) = 1;
  int n = s.i(I_NOBS, t);
  if (n == delta_t + 2) {              // the host appends and then drops the oldest beyond delta_t + 2
    for (int k = 1; k < n; ++k)
      for (int j = 0; j < 6; ++j) s.i(I_OBS + 6 * (k - 1) + j, t) = s.i(I_OBS + 6 * k + j, t);
    --n;
  }
  s.i(I_OBS + 6 * n, t) = age;
  for (int j = 0; j < 5; ++j) s.f(I_OBS + 6 * n + 1 + j, t) = r[j];
  s.i(I_NOBS, t) = n + 1;
  s.i(I_TSU, t) = 0;
  s.i(I_HITS, t) += 1;
  s.i(I_STREAK, t) += 1;
  ocs::Kalman kf;
  load_kf(s, t, kf);
  kf.update(ocs::box_to_z(r));
  store_kf(s, t, kf);
}

__device__ __noinline__ void new_track(const Tr& s, int t, const float* r, int id) {   // ocsort.py:275-281
  ocs::Kalman kf;
  const ocs::Meas z = ocs::box_to_z(r);
  for (int k = 0; k < 4; ++k) kf.x[k] = z.v[k];
  for (int i = 0; i < 7; ++i) kf.sx[i] = 0.;
  for (int i = 0; i < 49; ++i) kf.sP[i] = 0.;
  store_kf(s, t, kf);
  const int cls = static_cast<int>(r[5]);
  s.i(I_ID, t) = id;
  s.i(I_CLASS, t) = cls;
  s.f(I_SCORE, t) = r[4];
  s.i(I_NOCC, t) = 1;
  s.i(I_OCCL, t) = cls;
  s.f(I_OCC + cls, t) = 1.f;
  s.i(I_AGE, t) = 0;
  s.i(I_HITS, t) = 0;
  s.i(I_STREAK, t) = 0;
  s.i(I_TSU, t) = 0;
  s.i(I_HASLAST, t) = 0;
  for (int j = 0; j < 5; ++j) s.f(I_LAST + j, t) = 0.f;
  s.i(I_NOBS, t) = 0;
  for (int k = 0; k < 2; ++k) s.d(D_VEL + k, t) = s.d(D_AVG + k, t) = 0.;
  s.d(D_SPEED, t) = 0.;
}

// ocsort.py:143-155, plus what this frame reads before any update: the last observation and the cost's anchor
__device__ __noinline__ void track_predict(const Tr& s, int t, int delta_t) {
  ocs::Kalman kf;
  for (int i = 0; i < 7; ++i) kf.x[i] = s.d(D_X + i, t);
  for (int i = 0; i < 49; ++i) kf.P[i] = s.d(D_P + i, t);
  if (kf.x[6] + kf.x[2] <= 0.) kf.x[6] *= 0.;
  kf.predict();
  for (int i = 0; i < 7; ++i) s.d(D_X + i, t) = kf.x[i];
  for (int i = 0; i < 49; ++i) s.d(D_P + i, t) = kf.P[i];
  const int age = s.i(I_AGE, t) + 1;
  s.i(I_AGE, t) = age;
  if (s.i(I_TSU, t) > 0) s.i(I_STREAK, t) = 0;
  s.i(I_TSU, t) += 1;
  double box[4];
  ocs::state_to_box(kf.x, box);
  const bool hl = s.i(I_HASLAST, t);
  for (int k = 0; k < 4; ++k) {
    s.d(D_TRK + k, t) = box[k];
    s.d(D_LASTB + k, t) = hl ? static_cast<double>(s.f(I_LAST + k, t)) : -1.;
  }
  double pb[5] = {-1., -1., -1., -1., -1.};
  const int nobs = s.i(I_NOBS, t);
  if (nobs > 0) {
    int k = find_obs(s, t, age, delta_t);
    if (k < 0) k = nobs - 1;
    for (int j = 0; j < 5; ++j) pb[j] = s.f(I_OBS + 6 * k + 1 + j, t);
  }
  double valid, cx2, cy2;
  ocs::angle_anchor(pb, &valid, &cx2, &cy2);
  s.d(D_ANC, t) = valid;
  s.d(D_ANC + 1, t) = cx2;
  s.d(D_ANC + 2, t) = cy2;
  s.s(S_FLAGS, t) = 0;
}

// ------------------------------------------------------------------------------------------------- block helpers
struct Smem {
  int det[CC_OCSORT_MAX_ROWS];      // rows above the threshold, in row order
  int sec[CC_OCSORT_MAX_ROWS];      // rows of the BYTE band
  int udet[CC_OCSORT_MAX_ROWS];     // unmatched detections (indices into det)
  int2 cand[CC_OCSORT_MAX_ROWS];    // assignment result (row, column) in acceptance order
  double rmin[CC_OCSORT_MAX_ROWS];  // assignment: per-row minimum over the free columns ...
  int rcol[CC_OCSORT_MAX_ROWS];     // ... and its column
  char rflag[CC_OCSORT_MAX_ROWS];   // assignment: row used
  char cflag[CC_OCSORT_MAX_ROWS];   // first association: candidate fails the IoU filter
  char dflag[CC_OCSORT_MAX_ROWS];   // per detection: matched / listed / removed
  double wv[kWarps];
  long long wf[kWarps];
  int wc[kWarps];
  int bcast;
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


__device__ inline bool before(double v, long long f, double bv, long long bf) {   // (cost, flat index) order; bf < 0: none
  return f >= 0 && (bf < 0 || v < bv || (v == bv && f < bf));
}

// Minimum of row r over the free columns: the first one in column order among equal costs.
template <class Cost>
__device__ __noinline__ void row_min(Smem& sm, const Tr& s, int r, int C, const Cost& cost) {
  double best = 0.;
  int bc = -1;
  for (int c = 0; c < C; ++c) {
    if (s.s(S_COLUSED, c)) continue;
    const double v = cost(r, c);
    if (bc < 0 || v < best) { best = v; bc = c; }
  }
  sm.rmin[r] = best;
  sm.rcol[r] = bc;
}

// Greedy assignment (association.py:34-54) of R rows x C columns under cost(r, c): the pairs the host's walk over the
// (cost, flat index) order accepts, in its order, into sm.cand.  Returns their count, min(R, C).
template <class Cost>
__device__ int greedy(Smem& sm, const Tr& s, int R, int C, const Cost& cost) {
  for (int c = threadIdx.x; c < C; c += kThreads) s.s(S_COLUSED, c) = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < R; r += kThreads) {
    sm.rflag[r] = 0;
    row_min(sm, s, r, C, cost);
  }
  __syncthreads();
  const int K = R < C ? R : C;
  for (int k = 0; k < K; ++k) {
    double bv = 0.;
    long long bf = -1;
    for (int r = threadIdx.x; r < R; r += kThreads)
      if (!sm.rflag[r] && before(sm.rmin[r], static_cast<long long>(r) * C + sm.rcol[r], bv, bf)) {
        bv = sm.rmin[r];
        bf = static_cast<long long>(r) * C + sm.rcol[r];
      }
    for (int o = 16; o > 0; o >>= 1) {
      const double v = __shfl_down_sync(0xffffffffu, bv, o);
      const long long f = __shfl_down_sync(0xffffffffu, bf, o);
      if (before(v, f, bv, bf)) { bv = v; bf = f; }
    }
    if ((threadIdx.x & 31) == 0) {
      sm.wv[threadIdx.x >> 5] = bv;
      sm.wf[threadIdx.x >> 5] = bf;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kWarps; ++w)
        if (before(sm.wv[w], sm.wf[w], bv, bf)) { bv = sm.wv[w]; bf = sm.wf[w]; }
      const int r = static_cast<int>(bf / C), c = static_cast<int>(bf % C);
      sm.cand[k] = make_int2(r, c);
      sm.rflag[r] = 1;
      s.s(S_COLUSED, c) = 1;
      sm.bcast = c;
    }
    __syncthreads();
    const int c = sm.bcast;
    for (int r = threadIdx.x; r < R; r += kThreads)
      if (!sm.rflag[r] && sm.rcol[r] == c) row_min(sm, s, r, C, cost);
    __syncthreads();
  }
  return K;
}

// Moves the kept tracks (S_POS = new index, -1 = deleted) of [first, T) down in order, `G` lanes per round.
template <class V>
__device__ void compact_lanes(V* base, int cap, int lanes, const Tr& s, int first, int T) {
  constexpr int G = 8;
  for (int c0 = first; c0 < T; c0 += kThreads) {
    const int i = c0 + threadIdx.x;
    const int to = i < T ? s.s(S_POS, i) : -1;
    for (int l0 = 0; l0 < lanes; l0 += G) {
      V v[G];
#pragma unroll
      for (int g = 0; g < G; ++g)
        if (to >= 0 && l0 + g < lanes) v[g] = base[static_cast<size_t>(l0 + g) * cap + i];
      __syncthreads();
#pragma unroll
      for (int g = 0; g < G; ++g)
        if (to >= 0 && l0 + g < lanes) base[static_cast<size_t>(l0 + g) * cap + to] = v[g];
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------------- one camera per CTA
__global__ void __launch_bounds__(kThreads) ocsort_step_kernel(const __grid_constant__ JobTable jt, const SlotCfg* __restrict__ cfgs,
                                                               SlotCnt* __restrict__ cnts, int rb, double* __restrict__ out,
                                                               int cap_out, int* __restrict__ count, int* __restrict__ status) {
  __shared__ Smem sm;
  const cc_track_job job = jt.j[blockIdx.x];
  const SlotCfg cfg = cfgs[job.slot];
  const SlotCnt cnt = cnts[job.slot];
  const Tr s{cfg.dl, cfg.il, cfg.cap, lane_keep(rb)};
  const int T = cnt.T, n = job.n, delta_t = cfg.delta_t;
  const float thr = job.det_thresh;
  const float* rows = job.d_rows;
  const double th = cfg.iou_threshold;

  // ---- split the detections by threshold; class ids are checked before anything changes
  int D = 0, NS = 0;
  bool bad = false;
  for (int c0 = 0; c0 < n; c0 += kThreads) {
    const int i = c0 + threadIdx.x;
    const float sc = i < n ? rows[i * 6 + 4] : 0.f, cl = i < n ? rows[i * 6 + 5] : 0.f;
    const bool hi = i < n && sc > thr, lo = i < n && sc > 0.1f && sc < thr;
    if ((hi || lo) && !(cl >= 0.f && cl <= static_cast<float>(kClasses - 1) && cl == floorf(cl))) bad = true;
    const int ph = chunk_scan(sm, hi, &D);
    if (hi) sm.det[ph] = i;
    const int pl = chunk_scan(sm, lo, &NS);
    if (lo) sm.sec[pl] = i;
  }
  if (__syncthreads_or(bad)) {
    if (threadIdx.x == 0) { count[blockIdx.x] = 0; status[blockIdx.x] = CC_TRACK_BAD_CLASS; }
    return;
  }
  if (T + D > cfg.cap) {
    if (threadIdx.x == 0) { count[blockIdx.x] = T + D; status[blockIdx.x] = CC_TRACK_NEEDS_ROOM; }
    return;
  }
  const int frame_count = cnt.frame_count + 1;

  // ---- predict (ocsort.py:143-155); the cost's anchor and the last observation are read before any update
  for (int t = threadIdx.x; t < T; t += kThreads) track_predict(s, t, delta_t);
  __syncthreads();

  auto row = [&](int ri) { return rows + static_cast<size_t>(ri) * 6; };
  auto box4 = [&](int ri, double b[4]) {
    const float* r = row(ri);
    for (int k = 0; k < 4; ++k) b[k] = r[k];
  };
  auto lane4 = [&](int lane, int t, double b[4]) {
    for (int k = 0; k < 4; ++k) b[k] = s.d(lane + k, t);
  };
  auto iou_rt = [&](int ri, int lane, int t) {
    double a[4], b[4];
    box4(ri, a);
    lane4(lane, t, b);
    return ocs::iou(a, b);
  };

  // ---- first association (association.py:56-118)
  int ncand = 0, nud = 0, nut = 0;
  if (T == 0) {
    for (int d = threadIdx.x; d < D; d += kThreads) sm.udet[d] = d;
    nud = D;
  } else {
    if (D > 0) {
      bool gt1 = false, eq1 = false;
      for (int d = threadIdx.x; d < D; d += kThreads) {
        int rs = 0;
        for (int t = 0; t < T; ++t) rs += iou_rt(sm.det[d], D_TRK, t) > th;
        gt1 |= rs > 1;
        eq1 |= rs == 1;
      }
      for (int t = threadIdx.x; t < T; t += kThreads) {
        int cs = 0;
        for (int d = 0; d < D; ++d) cs += iou_rt(sm.det[d], D_TRK, t) > th;
        gt1 |= cs > 1;
      }
      const bool any_gt1 = __syncthreads_or(gt1), any_eq1 = __syncthreads_or(eq1);
      if (!any_gt1 && any_eq1) {             // max_row == max_col == 1: the pairs above the threshold, in row order
        for (int c0 = 0; c0 < D; c0 += kThreads) {
          const int d = c0 + threadIdx.x;
          int tt = -1;
          if (d < D)
            for (int t = 0; t < T && tt < 0; ++t)
              if (iou_rt(sm.det[d], D_TRK, t) > th) tt = t;
          const int p = chunk_scan(sm, tt >= 0, &ncand);
          if (tt >= 0) sm.cand[p] = make_int2(d, tt);
        }
      } else {                               // cost = -(IoU + velocity-direction consistency), ocsort.py:216-218
        const double inertia = cfg.inertia;
        ncand = greedy(sm, s, D, T, [&](int d, int t) {
          const int ri = sm.det[d];
          double a[4];
          box4(ri, a);
          const double vel[2] = {s.d(D_VEL, t), s.d(D_VEL + 1, t)};
          const double adc = ocs::angle_term(s.d(D_ANC, t), s.d(D_ANC + 1, t), s.d(D_ANC + 2, t), vel, a, row(ri)[4], inertia);
          return -(iou_rt(ri, D_TRK, t) + adc);
        });
      }
    }
    __syncthreads();
    for (int d = threadIdx.x; d < D; d += kThreads) sm.dflag[d] = 0;
    __syncthreads();
    for (int k = threadIdx.x; k < ncand; k += kThreads) {
      sm.dflag[sm.cand[k].x] = 1;
      s.s(S_FLAGS, sm.cand[k].y) = F_MATCHED;
      sm.cflag[k] = iou_rt(sm.det[sm.cand[k].x], D_TRK, sm.cand[k].y) < th;   // fails the IoU filter
    }
    __syncthreads();
    // unmatched: the unmatched indices in order, then the candidates that failed the filter, in candidate order
    for (int c0 = 0; c0 < D; c0 += kThreads) {
      const int d = c0 + threadIdx.x;
      const bool f = d < D && !sm.dflag[d];
      const int p = chunk_scan(sm, f, &nud);
      if (f) sm.udet[p] = d;
    }
    for (int c0 = 0; c0 < T; c0 += kThreads) {
      const int t = c0 + threadIdx.x;
      const bool f = t < T && !(s.s(S_FLAGS, t) & F_MATCHED);
      const int p = chunk_scan(sm, f, &nut);
      if (f) s.s(S_UTRK, p) = t;
    }
    for (int c0 = 0; c0 < ncand; c0 += kThreads) {
      const int k = c0 + threadIdx.x;
      const bool f = k < ncand && sm.cflag[k];
      int base = 0;
      const int p = chunk_scan(sm, f, &base);
      if (f) {
        sm.udet[nud + p] = sm.cand[k].x;
        s.s(S_UTRK, nut + p) = sm.cand[k].y;
      }
      nud += base;
      nut += base;
    }
    __syncthreads();
    // ---- updates of the matched tracks (each pair has its own track)
    for (int k = threadIdx.x; k < ncand; k += kThreads)
      if (!sm.cflag[k]) track_update(s, sm.cand[k].y, row(sm.det[sm.cand[k].x]), delta_t);
  }
  __syncthreads();

  // sorted_difference of un_trks (np.setdiff1d): the listed tracks not flagged F_REMOVED, ascending
  auto resort_trks = [&]() {
    for (int c = threadIdx.x; c < nut; c += kThreads) s.s(S_FLAGS, s.s(S_UTRK, c)) |= F_INUT;
    __syncthreads();
    int m = 0;
    for (int c0 = 0; c0 < T; c0 += kThreads) {
      const int t = c0 + threadIdx.x;
      const bool f = t < T && (s.s(S_FLAGS, t) & (F_INUT | F_REMOVED)) == F_INUT;
      const int p = chunk_scan(sm, f, &m);
      if (f) s.s(S_UTRK, p) = t;
    }
    nut = m;
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += kThreads) s.s(S_FLAGS, t) = 0;
    __syncthreads();
  };
  for (int t = threadIdx.x; t < T; t += kThreads) s.s(S_FLAGS, t) = 0;
  __syncthreads();

  // ---- BYTE: low-score detections against the still-unmatched predictions (ocsort.py:226-245)
  if (cfg.use_byte && NS > 0 && nut > 0) {
    bool any = false;
    for (int q = threadIdx.x; q < NS * nut; q += kThreads) any |= iou_rt(sm.sec[q / nut], D_TRK, s.s(S_UTRK, q % nut)) > th;
    if (__syncthreads_or(any)) {
      const int K = greedy(sm, s, NS, nut, [&](int r, int c) { return -iou_rt(sm.sec[r], D_TRK, s.s(S_UTRK, c)); });
      for (int k = threadIdx.x; k < K; k += kThreads) {
        const int ri = sm.sec[sm.cand[k].x], t = s.s(S_UTRK, sm.cand[k].y);
        if (iou_rt(ri, D_TRK, t) < th) continue;
        track_update(s, t, row(ri), delta_t);
        s.s(S_FLAGS, t) = F_REMOVED;
      }
      __syncthreads();
      resort_trks();
    }
  }
  // ---- observation-centric recovery: unmatched detections against last observations (ocsort.py:247-270)
  if (nud > 0 && nut > 0) {
    bool any = false;
    for (int q = threadIdx.x; q < nud * nut; q += kThreads) any |= iou_rt(sm.det[sm.udet[q / nut]], D_LASTB, s.s(S_UTRK, q % nut)) > th;
    if (__syncthreads_or(any)) {
      const int K = greedy(sm, s, nud, nut, [&](int r, int c) { return -iou_rt(sm.det[sm.udet[r]], D_LASTB, s.s(S_UTRK, c)); });
      for (int d = threadIdx.x; d < D; d += kThreads) sm.dflag[d] = 0;
      __syncthreads();
      for (int k = threadIdx.x; k < nud; k += kThreads) sm.dflag[sm.udet[k]] = F_INUT;
      __syncthreads();
      for (int k = threadIdx.x; k < K; k += kThreads) {
        const int d = sm.udet[sm.cand[k].x], t = s.s(S_UTRK, sm.cand[k].y);
        if (iou_rt(sm.det[d], D_LASTB, t) < th) continue;
        track_update(s, t, row(sm.det[d]), delta_t);
        s.s(S_FLAGS, t) = F_REMOVED;
        sm.dflag[d] |= F_REMOVED;
      }
      __syncthreads();
      int m = 0;
      for (int c0 = 0; c0 < D; c0 += kThreads) {
        const int d = c0 + threadIdx.x;
        const bool f = d < D && sm.dflag[d] == F_INUT;
        const int p = chunk_scan(sm, f, &m);
        if (f) sm.udet[p] = d;
      }
      nud = m;
      __syncthreads();
      resort_trks();
    }
  }
  for (int c = threadIdx.x; c < nut; c += kThreads) {
    track_none(s, s.s(S_UTRK, c));
  }
  // ---- new tracks, in the order of the unmatched list (ocsort.py:275-281)
  for (int k = threadIdx.x; k < nud; k += kThreads) new_track(s, T + k, row(sm.det[sm.udet[k]]), cnt.next_id + k);
  __syncthreads();

  // ---- output in reverse track order, then deletion (ocsort.py:282-302)
  const int T2 = T + nud;
  auto emits = [&](int t) {
    return s.i(I_TSU, t) < 1 && (s.i(I_STREAK, t) >= cfg.min_hits || frame_count <= cfg.min_hits);
  };
  int E = 0;
  for (int c0 = 0; c0 < T2; c0 += kThreads) {
    const int t = c0 + threadIdx.x;
    E += __syncthreads_count(t < T2 && emits(t));
  }
  double* o = out + static_cast<size_t>(blockIdx.x) * cap_out * 9;
  int e = 0, kept = 0;
  for (int c0 = 0; c0 < T2; c0 += kThreads) {
    const int t = c0 + threadIdx.x;
    const bool em = t < T2 && emits(t);
    const int p = chunk_scan(sm, em, &e);
    const int m = E - 1 - p;
    if (em && m < cap_out) {
      double d[4];
      if (!last_nonneg(s, t)) {
        double x[4];
        for (int k = 0; k < 4; ++k) x[k] = s.d(D_X + k, t);
        ocs::state_to_box(x, d);
      } else {
        for (int k = 0; k < 4; ++k) d[k] = s.f(I_LAST + k, t);
      }
      double* r = o + static_cast<size_t>(m) * 9;
      r[0] = d[0];
      r[1] = d[1];
      r[2] = d[2] - d[0];
      r[3] = d[3] - d[1];
      r[4] = s.f(I_SCORE, t);
      r[5] = s.i(I_CLASS, t);
      r[6] = s.i(I_ID, t) + 1;
      r[7] = s.i(I_AGE, t);
      r[8] = s.d(D_SPEED, t);
    }
    const int tsu = t < T2 ? s.i(I_TSU, t) : 0;
    const bool keep = t < T2 && !(tsu > cfg.max_age && (s.d(D_SPEED, t) > 2. || tsu > 600));
    const int q = chunk_scan(sm, keep, &kept);
    if (t < T2) s.s(S_POS, t) = keep ? q : -1;
  }
  if (kept < T2) {                     // order-preserving compaction from the first deleted track on
    if (threadIdx.x == 0) sm.bcast = T2;
    __syncthreads();
    for (int t = threadIdx.x; t < T2; t += kThreads)
      if (s.s(S_POS, t) < 0) atomicMin(&sm.bcast, t);
    __syncthreads();
    const int first = sm.bcast;
    compact_lanes(cfg.dl, cfg.cap, D_KEEP, s, first, T2);
    compact_lanes(cfg.il, cfg.cap, lane_keep(rb), s, first, T2);
  }
  if (threadIdx.x == 0) {
    cnts[job.slot] = SlotCnt{kept, frame_count, cnt.next_id + nud, 0};
    count[blockIdx.x] = E;
    status[blockIdx.x] = E > cap_out ? CC_TRACK_OVERFLOW : CC_TRACK_OK;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------- host side
namespace {

size_t track_bytes(const cc_ocsort_gpu* h) { return ND * sizeof(double) + static_cast<size_t>(lane_count(h->rb)) * 4; }

int alloc_slot(cc_ocsort_gpu* h, int cap, cudaStream_t st, SlotCfg& c) {
  void* p = nullptr;
  CC_CHECK_CUDA(cudaMallocAsync(&p, static_cast<size_t>(cap) * track_bytes(h), st));
  c.dl = static_cast<double*>(p);
  c.il = reinterpret_cast<int32_t*>(static_cast<char*>(p) + static_cast<size_t>(cap) * ND * sizeof(double));
  c.cap = cap;
  return CC_OK;
}

int push_cfg(cc_ocsort_gpu* h, int slot, cudaStream_t st) {
  CC_CHECK_CUDA(cudaMemcpyAsync(h->d_cfg + slot, &h->cfg[slot], sizeof(SlotCfg), cudaMemcpyHostToDevice, st));
  return CC_OK;
}

}  // namespace

extern "C" {

int cc_ocsort_gpu_create(int slots, int max_delta_t, cc_ocsort_gpu** out) {
  CC_REQUIRE(out && slots > 0 && slots <= (1 << 20) && max_delta_t >= 1 && max_delta_t <= 64,
             "cc_ocsort_gpu_create: bad arguments (slots %d, max_delta_t %d)", slots, max_delta_t);
  cc_ocsort_gpu* h = new cc_ocsort_gpu();
  h->S = slots;
  h->rb = max_delta_t + 2;
  h->cfg.assign(slots, SlotCfg{});
  cudaError_t e = cudaMalloc(&h->d_cfg, sizeof(SlotCfg) * slots);
  if (e == cudaSuccess) e = cudaMalloc(&h->d_cnt, sizeof(SlotCnt) * slots);
  if (e == cudaSuccess) e = cudaMemset(h->d_cfg, 0, sizeof(SlotCfg) * slots);
  if (e == cudaSuccess) e = cudaMemset(h->d_cnt, 0, sizeof(SlotCnt) * slots);
  if (e != cudaSuccess) {
    cudaFree(h->d_cfg);
    cudaFree(h->d_cnt);
    delete h;
    cc::set_error("cc_ocsort_gpu_create: %s", cudaGetErrorString(e));
    return cc::CC_ERR_CUDA;
  }
  *out = h;
  return CC_OK;
}

int cc_ocsort_gpu_destroy(cc_ocsort_gpu* h) {
  if (!h) return CC_OK;
  cudaDeviceSynchronize();            // slot storage is freed stream-ordered elsewhere; here nothing may still use it
  cc_events_destroy(h);
  cc_alerts_destroy(h);
  for (auto& c : h->cfg)
    if (c.active) cudaFree(c.dl);
  cudaFree(h->d_cfg);
  cudaFree(h->d_cnt);
  delete h;
  return CC_OK;
}

int cc_ocsort_gpu_configure(cc_ocsort_gpu* h, int slot, int max_age, int min_hits, double iou_threshold, int delta_t,
                            double inertia, int use_byte, int capacity, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S, "cc_ocsort_gpu_configure: bad handle or slot %d", slot);
  CC_REQUIRE(max_age >= 0 && min_hits >= 0 && delta_t >= 1 && capacity >= 1 && capacity <= (1 << 20),
             "cc_ocsort_gpu_configure: bad arguments");
  CC_REQUIRE(delta_t + 2 <= h->rb, "cc_ocsort_gpu_configure: delta_t %d exceeds the handle's bound %d", delta_t, h->rb - 2);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  SlotCfg& c = h->cfg[slot];
  if (c.active && c.cap != capacity) {
    CC_CHECK_CUDA(cudaFreeAsync(c.dl, st));
    c.active = 0;
  }
  if (!c.active) {
    const int r = alloc_slot(h, capacity, st, c);
    if (r != CC_OK) return r;
  }
  c.active = 1;
  c.max_age = max_age;
  c.min_hits = min_hits;
  c.delta_t = delta_t;
  c.use_byte = use_byte ? 1 : 0;
  c.iou_threshold = iou_threshold;
  c.inertia = inertia;
  CC_CHECK_CUDA(cudaMemsetAsync(h->d_cnt + slot, 0, sizeof(SlotCnt), st));
  int r = cc_events_slot_clear(h, slot, st);   // a restarted tracker reuses ids: its events start afresh too
  if (r != CC_OK) return r;
  r = cc_alerts_slot_clear(h, slot, st);       // and, as init_cam, its object counter and alert warm-up
  if (r != CC_OK) return r;
  return push_cfg(h, slot, st);
}

int cc_ocsort_gpu_free(cc_ocsort_gpu* h, int slot, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S, "cc_ocsort_gpu_free: bad handle or slot %d", slot);
  SlotCfg& c = h->cfg[slot];
  if (!c.active) return CC_OK;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int r = cc_events_slot_free(h, slot, st);
  if (r != CC_OK) return r;
  r = cc_alerts_slot_free(h, slot, st);
  if (r != CC_OK) return r;
  CC_CHECK_CUDA(cudaFreeAsync(c.dl, st));
  c = SlotCfg{};
  return push_cfg(h, slot, st);
}

int cc_ocsort_gpu_grow(cc_ocsort_gpu* h, int slot, int capacity, void* stream) {
  CC_REQUIRE(h && slot >= 0 && slot < h->S && h->cfg[slot].active, "cc_ocsort_gpu_grow: bad handle or slot %d", slot);
  SlotCfg& c = h->cfg[slot];
  CC_REQUIRE(capacity <= (1 << 20), "cc_ocsort_gpu_grow: capacity %d too large", capacity);
  if (capacity <= c.cap) return CC_OK;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  SlotCfg n = c;
  const int r = alloc_slot(h, capacity, st, n);
  if (r != CC_OK) return r;
  // every lane keeps its first c.cap entries: one strided copy per region
  CC_CHECK_CUDA(cudaMemcpy2DAsync(n.dl, n.cap * sizeof(double), c.dl, c.cap * sizeof(double), c.cap * sizeof(double), ND,
                                  cudaMemcpyDeviceToDevice, st));
  CC_CHECK_CUDA(cudaMemcpy2DAsync(n.il, n.cap * 4, c.il, c.cap * 4, c.cap * 4, lane_count(h->rb), cudaMemcpyDeviceToDevice, st));
  CC_CHECK_CUDA(cudaFreeAsync(c.dl, st));
  c = n;
  return push_cfg(h, slot, st);
}

int cc_ocsort_gpu_capacity(cc_ocsort_gpu* h, int slot, int* capacity) {
  CC_REQUIRE(h && capacity && slot >= 0 && slot < h->S, "cc_ocsort_gpu_capacity: bad arguments");
  *capacity = h->cfg[slot].active ? h->cfg[slot].cap : 0;
  return CC_OK;
}

int cc_ocsort_gpu_num_tracks(cc_ocsort_gpu* h, int slot, int* n, void* stream) {
  CC_REQUIRE(h && n && slot >= 0 && slot < h->S, "cc_ocsort_gpu_num_tracks: bad arguments");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  SlotCnt c;
  CC_CHECK_CUDA(cudaMemcpyAsync(&c, h->d_cnt + slot, sizeof c, cudaMemcpyDeviceToHost, st));   // after the stream's updates
  CC_CHECK_CUDA(cudaStreamSynchronize(st));
  *n = h->cfg[slot].active ? c.T : 0;
  return CC_OK;
}

int cc_ocsort_gpu_update(cc_ocsort_gpu* h, const cc_track_job* jobs, int B, double* d_out, int cap, int* d_count,
                         int* d_status, void* stream) {
  CC_REQUIRE(h && jobs && d_out && d_count && d_status && B >= 1 && B <= CC_MAX_FRAMES && cap >= 0,
             "cc_ocsort_gpu_update: bad arguments (B %d, cap %d)", B, cap);
  static thread_local std::vector<char> seen;
  seen.assign(h->S, 0);
  JobTable jt;
  for (int b = 0; b < B; ++b) {
    const cc_track_job& j = jobs[b];
    CC_REQUIRE(j.slot >= 0 && j.slot < h->S && h->cfg[j.slot].active, "cc_ocsort_gpu_update: job %d: slot %d is not configured", b,
               j.slot);
    CC_REQUIRE(!seen[j.slot], "cc_ocsort_gpu_update: job %d: slot %d appears twice", b, j.slot);
    CC_REQUIRE(j.n >= 0 && j.n <= CC_OCSORT_MAX_ROWS && (j.d_rows || j.n == 0),
               "cc_ocsort_gpu_update: job %d: %d rows at %p (0..%d rows, non-null)", b, j.n, static_cast<const void*>(j.d_rows),
               CC_OCSORT_MAX_ROWS);
    seen[j.slot] = 1;
    jt.j[b] = j;
  }
  ocsort_step_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(jt, h->d_cfg, h->d_cnt, h->rb, d_out, cap, d_count,
                                                                              d_status);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // extern "C"
