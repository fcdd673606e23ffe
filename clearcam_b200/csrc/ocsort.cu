// Observation-centric SORT tracker, the consumer of the detector's (B,300,6) rows (SURVEY.md §8f N2).
//
// Host C++ (no device code; the file is .cu only so the one Makefile rule builds it).  The reference runs this per camera
// in numpy at ~6 ms/frame (ocsort_tracker/ocsort.py:163-308, association.py, kalmanfilter.py); behind a detector that
// delivers thousands of frames/s that is the bottleneck, so it is rebuilt here as flat-array C++ (a few microseconds
// per frame) behind cc_ocsort_* and checked against golden vectors produced by the reference itself
// (tests/golden/ocsort_*.npz, oracle/make_golden_ocsort.py).  The per-track arithmetic (filter, boxes, IoU, direction,
// angle cost) lives in ocsort_math.cuh, shared with the device tracker of ocsort_gpu.cu, which is held to this one bit
// for bit; this file keeps the control flow.
//
// Arithmetic follows the reference's dtypes where they reach the state: detector rows are float32 and the reference
// converts a box to the filter measurement, the track direction and the mean speed in float32 before anything is
// promoted to float64 (ocsort.py:21-33, 48-53, 123-125); the filter itself is float64.  Association costs are computed
// in float64 (the reference's dtype there depends on which tracks exist; only exact ties could tell the difference).
#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>
#include <numeric>
#include <thread>
#include <vector>

#include "cc_common.h"
#include "clearcam_b200.h"
#include "ocsort_math.cuh"

using cc::CC_ERR_INVALID;
using cc::CC_OK;

namespace {

using ocs::Kalman;
using ocs::Meas;
using ocs::box_to_z;
using ocs::iou;
using ocs::state_to_box;

// ------------------------------------------------------------------------------------------------- one track
struct Obs { float b[5]; };

struct Track {
  Kalman kf;
  int id = 0, age = 0, hits = 0, hit_streak = 0, time_since_update = 0;
  bool has_last = false;                 // false: the reference's [-1,-1,-1,-1,-1] placeholder (ocsort.py:98)
  Obs last{};
  std::vector<std::pair<int, Obs>> obs;  // (age, observation): only the last delta_t+1 can ever be looked up
  double vel[2] = {0., 0.};              // unit direction (dy, dx)
  double avg_vel[2] = {0., 0.};
  double speed = 0.;
  std::vector<std::pair<int, float>> occ;   // class -> accumulated score, insertion-ordered like the dict
  int class_id = 0;
  float score = 0.f;

  // `last_observation.sum() >= 0` (ocsort.py:113, 281): a real box whose five numbers sum below zero reads as "none"
  bool last_nonneg() const {
    return has_last && ocs::box_sum_nonneg(last.b);
  }
  const Obs* find_obs(int a) const {
    for (auto it = obs.rbegin(); it != obs.rend(); ++it)
      if (it->first == a) return &it->second;
    return nullptr;
  }
};

// association.py:34-54: walk the pairs by ascending cost, take a pair when its row and column are both free, stop when
// every row or every column is used.  Ties are broken by flat index (the reference's argsort leaves them unspecified).
static void greedy_assign(const std::vector<double>& cost, int rows, int cols, std::vector<std::array<int, 2>>& out) {
  out.clear();
  if (rows == 0 || cols == 0) return;
  // The walk usually ends after min(rows, cols) good pairs, so a heap (O(n) to build, O(log n) per pair looked at)
  // replaces the reference's full argsort.  Order = (cost, flat index) ascending.
  typedef std::pair<double, int> E;
  std::vector<E> heap(static_cast<size_t>(rows) * cols);
  for (size_t i = 0; i < heap.size(); ++i) heap[i] = E(cost[i], static_cast<int>(i));
  auto later = [](const E& a, const E& b) { return a.first > b.first || (a.first == b.first && a.second > b.second); };
  std::make_heap(heap.begin(), heap.end(), later);
  std::vector<char> ru(rows, 0), cu(cols, 0);
  int nr = 0, nc = 0;
  auto end = heap.end();
  while (end != heap.begin()) {
    std::pop_heap(heap.begin(), end, later);
    --end;
    const int f = end->second, r = f / cols, c = f % cols;
    if (ru[r] || cu[c]) continue;
    out.push_back({r, c});
    ru[r] = cu[c] = 1;
    ++nr;
    ++nc;
    if (nr == rows || nc == cols) break;
  }
}

static void sorted_difference(std::vector<int>& a, const std::vector<int>& remove) {   // np.setdiff1d
  std::sort(a.begin(), a.end());
  a.erase(std::unique(a.begin(), a.end()), a.end());
  a.erase(std::remove_if(a.begin(), a.end(), [&](int v) { return std::find(remove.begin(), remove.end(), v) != remove.end(); }),
          a.end());
}

}  // namespace

// ------------------------------------------------------------------------------------------------- the tracker
struct cc_ocsort {
  int max_age, min_hits, delta_t, use_byte;
  double iou_threshold, inertia;
  int frame_count = 0, next_id = 0;
  std::vector<std::unique_ptr<Track>> trackers;

  // ---- per-track steps
  void track_predict(Track& t, double box[4]) {   // ocsort.py:143-155
    if (t.kf.x[6] + t.kf.x[2] <= 0.) t.kf.x[6] *= 0.;
    t.kf.predict();
    t.age += 1;
    if (t.time_since_update > 0) t.hit_streak = 0;
    t.time_since_update += 1;
    state_to_box(t.kf.x, box);
  }

  void track_update(Track& t, const float* b, float score, int cls) {   // ocsort.py:105-139, bbox present
    auto it = std::find_if(t.occ.begin(), t.occ.end(), [&](const std::pair<int, float>& p) { return p.first == cls; });
    if (it == t.occ.end()) t.occ.push_back({cls, score});
    else it->second += score;
    float best = t.occ[0].second;
    t.class_id = t.occ[0].first;
    for (auto& p : t.occ)
      if (p.second > best) { best = p.second; t.class_id = p.first; }
    if (t.last_nonneg()) {
      const Obs* prev = nullptr;
      for (int i = 0; i < delta_t && !prev; ++i) prev = t.find_obs(t.age - (delta_t - i));
      if (!prev) prev = &t.last;
      ocs::velocity_update(prev->b, b, t.age, t.vel, t.avg_vel, &t.speed);
    }
    std::memcpy(t.last.b, b, sizeof t.last.b);
    t.has_last = true;
    t.obs.push_back({t.age, t.last});
    if (static_cast<int>(t.obs.size()) > delta_t + 2) t.obs.erase(t.obs.begin());
    t.time_since_update = 0;
    t.hits += 1;
    t.hit_streak += 1;
    t.kf.update(box_to_z(b));
  }

  // ---- one frame (ocsort.py:177-308)
  int update(const float* rows, int n, float det_thresh, double* out, int cap, int* n_out) {
    frame_count += 1;
    struct Det { float b[5]; int cls; };
    std::vector<Det> dets, second;
    for (int i = 0; i < n; ++i) {
      const float* r = rows + static_cast<size_t>(i) * 6;
      Det d;
      std::memcpy(d.b, r, 5 * sizeof(float));
      d.cls = static_cast<int>(r[5]);
      if (r[4] > 0.1f && r[4] < det_thresh) second.push_back(d);
      if (r[4] > det_thresh) dets.push_back(d);
    }
    const int D = static_cast<int>(dets.size()), T = static_cast<int>(trackers.size());

    std::vector<std::array<double, 4>> trks(T);
    for (int t = 0; t < T; ++t) track_predict(*trackers[t], trks[t].data());

    // ---- first association (association.py:56-118)
    std::vector<std::array<int, 2>> matched;          // (det, trk), IoU-filtered
    std::vector<int> un_dets, un_trks;
    std::vector<double> iou_m(static_cast<size_t>(D) * T);
    if (T == 0) {
      for (int d = 0; d < D; ++d) un_dets.push_back(d);
    } else {
      std::vector<std::array<double, 4>> dbox(D);
      for (int d = 0; d < D; ++d)
        for (int k = 0; k < 4; ++k) dbox[d][k] = dets[d].b[k];
      for (int d = 0; d < D; ++d)
        for (int t = 0; t < T; ++t) iou_m[static_cast<size_t>(d) * T + t] = iou(dbox[d].data(), trks[t].data());
      std::vector<std::array<int, 2>> cand;
      if (D > 0) {
        int max_row = 0, max_col = 0;
        std::vector<int> colsum(T, 0);
        for (int d = 0; d < D; ++d) {
          int rs = 0;
          for (int t = 0; t < T; ++t)
            if (iou_m[static_cast<size_t>(d) * T + t] > iou_threshold) { ++rs; ++colsum[t]; }
          max_row = std::max(max_row, rs);
        }
        for (int t = 0; t < T; ++t) max_col = std::max(max_col, colsum[t]);
        if (max_row == 1 && max_col == 1) {
          for (int d = 0; d < D; ++d)
            for (int t = 0; t < T; ++t)
              if (iou_m[static_cast<size_t>(d) * T + t] > iou_threshold) cand.push_back({d, t});
        } else {
          // cost = -(IoU + velocity-direction consistency), ocsort.py:216-218 / association.py:60-82
          std::vector<double> cost(static_cast<size_t>(D) * T);
          for (int t = 0; t < T; ++t) {
            const Track& tr = *trackers[t];
            // observation delta_t frames back (ocsort.py:11-19)
            const Obs* ko = nullptr;
            if (!tr.obs.empty()) {
              for (int i = 0; i < delta_t && !ko; ++i) ko = tr.find_obs(tr.age - (delta_t - i));
              if (!ko) ko = &tr.obs.back().second;
            }
            const double pb[5] = {ko ? ko->b[0] : -1., ko ? ko->b[1] : -1., ko ? ko->b[2] : -1., ko ? ko->b[3] : -1., ko ? ko->b[4] : -1.};
            double valid, cx2, cy2;
            ocs::angle_anchor(pb, &valid, &cx2, &cy2);
            for (int d = 0; d < D; ++d) {
              const double adc = ocs::angle_term(valid, cx2, cy2, tr.vel, dbox[d].data(), dets[d].b[4], inertia);
              cost[static_cast<size_t>(d) * T + t] = -(iou_m[static_cast<size_t>(d) * T + t] + adc);
            }
          }
          greedy_assign(cost, D, T, cand);
        }
      }
      std::vector<char> dm(D, 0), tm(T, 0);
      for (auto& m : cand) dm[m[0]] = tm[m[1]] = 1;
      for (int d = 0; d < D; ++d)
        if (!dm[d]) un_dets.push_back(d);
      for (int t = 0; t < T; ++t)
        if (!tm[t]) un_trks.push_back(t);
      for (auto& m : cand) {
        if (iou_m[static_cast<size_t>(m[0]) * T + m[1]] < iou_threshold) {
          un_dets.push_back(m[0]);
          un_trks.push_back(m[1]);
        } else {
          matched.push_back(m);
        }
      }
    }
    // last observations are read before this frame's updates (ocsort.py:207)
    std::vector<std::array<double, 4>> last_boxes(T);
    for (int t = 0; t < T; ++t)
      for (int k = 0; k < 4; ++k) last_boxes[t][k] = trackers[t]->has_last ? trackers[t]->last.b[k] : -1.;
    for (auto& m : matched) track_update(*trackers[m[1]], dets[m[0]].b, dets[m[0]].b[4], dets[m[0]].cls);

    std::vector<std::array<int, 2>> re;
    // ---- BYTE: low-score detections against still-unmatched predictions (ocsort.py:226-245)
    if (use_byte && !second.empty() && !un_trks.empty()) {
      const int R = static_cast<int>(second.size()), C = static_cast<int>(un_trks.size());
      std::vector<double> io(static_cast<size_t>(R) * C), neg(static_cast<size_t>(R) * C);
      double mx = -INFINITY;
      for (int r = 0; r < R; ++r) {
        const double b[4] = {second[r].b[0], second[r].b[1], second[r].b[2], second[r].b[3]};
        for (int c = 0; c < C; ++c) {
          const double v = iou(b, trks[un_trks[c]].data());
          io[static_cast<size_t>(r) * C + c] = v;
          neg[static_cast<size_t>(r) * C + c] = -v;
          mx = std::max(mx, v);
        }
      }
      if (mx > iou_threshold) {
        greedy_assign(neg, R, C, re);
        std::vector<int> rm;
        for (auto& m : re) {
          if (io[static_cast<size_t>(m[0]) * C + m[1]] < iou_threshold) continue;
          const int ti = un_trks[m[1]];
          track_update(*trackers[ti], second[m[0]].b, second[m[0]].b[4], second[m[0]].cls);
          rm.push_back(ti);
        }
        sorted_difference(un_trks, rm);
      }
    }
    // ---- observation-centric recovery: unmatched detections against last observations (ocsort.py:247-270)
    if (!un_dets.empty() && !un_trks.empty()) {
      const int R = static_cast<int>(un_dets.size()), C = static_cast<int>(un_trks.size());
      std::vector<double> io(static_cast<size_t>(R) * C), neg(static_cast<size_t>(R) * C);
      double mx = -INFINITY;
      for (int r = 0; r < R; ++r) {
        const Det& dd = dets[un_dets[r]];
        const double b[4] = {dd.b[0], dd.b[1], dd.b[2], dd.b[3]};
        for (int c = 0; c < C; ++c) {
          const double v = iou(b, last_boxes[un_trks[c]].data());
          io[static_cast<size_t>(r) * C + c] = v;
          neg[static_cast<size_t>(r) * C + c] = -v;
          mx = std::max(mx, v);
        }
      }
      if (mx > iou_threshold) {
        greedy_assign(neg, R, C, re);
        std::vector<int> rmd, rmt;
        for (auto& m : re) {
          if (io[static_cast<size_t>(m[0]) * C + m[1]] < iou_threshold) continue;
          const int di = un_dets[m[0]], ti = un_trks[m[1]];
          track_update(*trackers[ti], dets[di].b, dets[di].b[4], dets[di].cls);
          rmd.push_back(di);
          rmt.push_back(ti);
        }
        sorted_difference(un_dets, rmd);
        sorted_difference(un_trks, rmt);
      }
    }
    for (int t : un_trks) trackers[t]->kf.update_none();

    for (int d : un_dets) {                              // ocsort.py:275-281
      std::unique_ptr<Track> t(new Track());
      const Meas z = box_to_z(dets[d].b);
      for (int k = 0; k < 4; ++k) t->kf.x[k] = z.v[k];
      t->id = next_id++;
      t->class_id = dets[d].cls;
      t->score = dets[d].b[4];
      t->occ.push_back({dets[d].cls, 1.f});
      trackers.push_back(std::move(t));
    }

    int m = 0;
    for (int i = static_cast<int>(trackers.size()) - 1; i >= 0; --i) {      // ocsort.py:282-302
      Track& t = *trackers[i];
      double d[4];
      if (!t.last_nonneg()) {
        state_to_box(t.kf.x, d);
      } else {
        for (int k = 0; k < 4; ++k) d[k] = t.last.b[k];
      }
      if (t.time_since_update < 1 && (t.hit_streak >= min_hits || frame_count <= min_hits)) {
        if (m < cap) {
          double* o = out + static_cast<size_t>(m) * 9;
          o[0] = d[0];
          o[1] = d[1];
          o[2] = d[2] - d[0];
          o[3] = d[3] - d[1];
          o[4] = t.score;
          o[5] = t.class_id;
          o[6] = t.id + 1;
          o[7] = t.age;
          o[8] = t.speed;
        }
        ++m;
      }
      if (t.time_since_update > max_age && (t.speed > 2. || t.time_since_update > 600)) trackers.erase(trackers.begin() + i);
    }
    *n_out = m;
    if (m > cap) {
      cc::set_error("cc_ocsort_update: %d tracks do not fit the output capacity %d", m, cap);
      return CC_ERR_INVALID;
    }
    return CC_OK;
  }
};

extern "C" {

int cc_ocsort_create(int max_age, int min_hits, double iou_threshold, int delta_t, double inertia, int use_byte, cc_ocsort_t* out) {
  if (!out || max_age < 0 || min_hits < 0 || delta_t < 1) {
    cc::set_error("cc_ocsort_create: bad arguments");
    return CC_ERR_INVALID;
  }
  cc_ocsort* h = new cc_ocsort();
  h->max_age = max_age;
  h->min_hits = min_hits;
  h->iou_threshold = iou_threshold;
  h->delta_t = delta_t;
  h->inertia = inertia;
  h->use_byte = use_byte;
  *out = h;
  return CC_OK;
}

int cc_ocsort_destroy(cc_ocsort_t h) {
  delete h;
  return CC_OK;
}

int cc_ocsort_update(cc_ocsort_t h, const float* rows, int n, float det_thresh, double* out, int cap, int* n_out) {
  if (!h || (!rows && n > 0) || !out || !n_out || n < 0 || cap < 0) {
    cc::set_error("cc_ocsort_update: bad arguments");
    return CC_ERR_INVALID;
  }
  return h->update(rows, n, det_thresh, out, cap, n_out);
}

int cc_ocsort_update_batch(cc_ocsort_t* hs, int B, const float* rows, int n, const float* det_thresh, double* out, int cap,
                           int* n_out) {
  if (!hs || !rows || !det_thresh || !out || !n_out || B < 0) {
    cc::set_error("cc_ocsort_update_batch: bad arguments");
    return CC_ERR_INVALID;
  }
  // cameras are independent: split them over a few host threads when there are enough to pay for the spawn
  std::atomic<int> next(0), bad(0);
  auto work = [&]() {
    for (int b = next.fetch_add(1); b < B; b = next.fetch_add(1)) {
      if (!hs[b]) { n_out[b] = 0; continue; }
      const int r = hs[b]->update(rows + static_cast<size_t>(b) * n * 6, n, det_thresh[b], out + static_cast<size_t>(b) * cap * 9,
                                  cap, n_out + b);
      if (r != CC_OK) bad.store(1);
    }
  };
  const int hw = static_cast<int>(std::thread::hardware_concurrency());
  const int nthr = std::max(1, std::min({B / 4, hw > 0 ? hw : 1, 16}));
  if (nthr <= 1) {
    work();
  } else {
    std::vector<std::thread> pool;
    for (int i = 1; i < nthr; ++i) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
  }
  if (bad.load()) {
    cc::set_error("cc_ocsort_update_batch: a camera produced more tracks than the output capacity %d", cap);
    return CC_ERR_INVALID;
  }
  return CC_OK;
}

int cc_ocsort_num_tracks(cc_ocsort_t h) { return h ? static_cast<int>(h->trackers.size()) : 0; }

}  // extern "C"
