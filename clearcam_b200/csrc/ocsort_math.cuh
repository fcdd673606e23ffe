// Per-track arithmetic of the OC-SORT tracker, shared by the host tracker (ocsort.cu) and the device tracker
// (ocsort_gpu.cu) so that both run the very same operations in the very same order.  Every function is
// __host__ __device__; the device file is built with -fmad=false (no contraction) and without fast-math, so float32 steps
// stay float32, division and sqrt stay IEEE and the only libm call whose bits may differ between the two sides is acos
// (angle_term).  Comparisons are written as std::max / std::min evaluate them (a < b ? b : a), not fmax / fmin.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define OCS_HD __host__ __device__ __forceinline__
#define OCS_HD_CALL __host__ __device__ __noinline__   // the filter's heavy steps: one copy each, own frame
#else
#define OCS_HD inline
#define OCS_HD_CALL inline
#endif
// Keeps a device loop rolled (the filter's 7x7 products would otherwise be held in registers and spill); no effect on
// the order of any operation.
#ifdef __CUDA_ARCH__
#define OCS_ROLLED _Pragma("unroll 1")
#else
#define OCS_ROLLED
#endif

namespace ocs {

OCS_HD double dmax(double a, double b) { return a < b ? b : a; }   // std::max
OCS_HD double dmin(double a, double b) { return b < a ? b : a; }   // std::min

// 7-state constant-velocity filter on z = [cx, cy, area, aspect] (ocsort.py:69-80): F = I + shift(4), H = [I4 0],
// R = diag(1,1,10,10), P0 = diag(10,10,10,10,1e4,1e4,1e4), Q = diag(1,1,1,1,.01,.01,1e-4).
OCS_HD double kR(int i) { return i < 2 ? 1. : 10.; }
OCS_HD double kQ(int i) { return i < 4 ? 1. : i < 6 ? 0.01 : 0.0001; }

struct Meas {
  bool some = false;   // false = "no observation this frame"
  bool f32 = false;    // the four numbers were produced by float32 arithmetic (a real detection) rather than float64
  double v[4] = {0, 0, 0, 0};
};

OCS_HD bool invert4(const double S[16], double inv[16]) {
  double a[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      a[i][j] = S[i * 4 + j];
      a[i][4 + j] = i == j ? 1. : 0.;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r)
      if (fabs(a[r][c]) > fabs(a[piv][c])) piv = r;
    if (a[piv][c] == 0.) return false;
    if (piv != c)
      for (int j = 0; j < 8; ++j) {
        const double t = a[piv][j];
        a[piv][j] = a[c][j];
        a[c][j] = t;
      }
    const double d = 1. / a[c][c];
    for (int j = 0; j < 8; ++j) a[c][j] *= d;
    for (int r = 0; r < 4; ++r) {
      if (r == c) continue;
      const double f = a[r][c];
      if (f != 0.)
        for (int j = 0; j < 8; ++j) a[r][j] -= f * a[c][j];
    }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) inv[i * 4 + j] = a[i][4 + j];
  return true;
}

// The reference appends every measurement (or None) to a list that only ever answers one question: where are the last two
// real entries (kalmanfilter.py:57, 70-74).  Keeping just those and the length is equivalent and does not grow.
struct History {
  int len = 0;
  int idx[2] = {-1, -1};     // [0] = last real entry, [1] = the one before
  Meas m[2];
  OCS_HD void push(const Meas& z) {
    if (z.some) {
      idx[1] = idx[0];
      m[1] = m[0];
      idx[0] = len;
      m[0] = z;
    }
    ++len;
  }
};

struct Kalman {
  double x[7];
  double P[49];
  History hist;
  bool observed = false;
  // state frozen when the track was last seen (kalmanfilter.py:112-114); restored by the re-update on re-acquisition
  bool has_saved = false;
  double sx[7];
  double sP[49];
  History shist;

  OCS_HD Kalman() {
    for (int i = 0; i < 7; ++i) x[i] = 0.;
    for (int i = 0; i < 49; ++i) P[i] = 0.;
    for (int i = 0; i < 7; ++i) P[i * 7 + i] = i < 4 ? 10. : 10000.;
  }

  OCS_HD void predict() {            // kalmanfilter.py:65-67
    double FP[49];
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 7; ++j) FP[i * 7 + j] = i < 3 ? P[i * 7 + j] + P[(i + 4) * 7 + j] : P[i * 7 + j];
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 7; ++j) P[i * 7 + j] = (j < 3 ? FP[i * 7 + j] + FP[i * 7 + j + 4] : FP[i * 7 + j]) + (i == j ? kQ(i) : 0.);
    x[0] += x[4];
    x[1] += x[5];
    x[2] += x[6];
  }

  OCS_HD_CALL void correct(const double z[4]) {   // kalmanfilter.py:121-131 (Joseph form)
    double y[4], S[16], SI[16], K[28];
    for (int i = 0; i < 4; ++i) y[i] = z[i] - x[i];
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) S[i * 4 + j] = P[i * 7 + j] + (i == j ? kR(i) : 0.);
    if (!invert4(S, SI)) return;
    OCS_ROLLED
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 4; ++j) {
        double s = 0.;
        for (int k = 0; k < 4; ++k) s += P[i * 7 + k] * SI[k * 4 + j];
        K[i * 4 + j] = s;
      }
    for (int i = 0; i < 7; ++i) {
      double s = 0.;
      for (int k = 0; k < 4; ++k) s += K[i * 4 + k] * y[k];
      x[i] += s;
    }
    double A[49], AP[49];       // A = I - K H
    OCS_ROLLED
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 7; ++j) A[i * 7 + j] = (i == j ? 1. : 0.) - (j < 4 ? K[i * 4 + j] : 0.);
    OCS_ROLLED
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 7; ++j) {
        double s = 0.;
        for (int k = 0; k < 7; ++k) s += A[i * 7 + k] * P[k * 7 + j];
        AP[i * 7 + j] = s;
      }
    OCS_ROLLED
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 7; ++j) {
        double s = 0.;
        for (int k = 0; k < 7; ++k) s += AP[i * 7 + k] * A[j * 7 + k];
        double krk = 0.;
        for (int k = 0; k < 4; ++k) krk += K[i * 4 + k] * kR(k) * K[j * 4 + k];
        P[i * 7 + j] = s + krk;      // AP holds everything P is still needed for
      }
  }

  OCS_HD void update_none() {        // kalmanfilter.py:109-117
    hist.push(Meas{});
    if (observed) {
      has_saved = true;
      for (int i = 0; i < 7; ++i) sx[i] = x[i];
      for (int i = 0; i < 49; ++i) sP[i] = P[i];
      shist = hist;
    }
    observed = false;
  }

  // Observation-centric re-update (kalmanfilter.py:69-105): roll back to the frozen state and replay a straight-line
  // virtual trajectory from the last observation before the gap to the new one.
  OCS_HD_CALL void unfreeze() {
    const int i2 = hist.idx[0], i1 = hist.idx[1];
    if (i1 < 0) return;
    const Meas a = hist.m[1], b = hist.m[0];
    // float32 where the reference's operands are both float32 (two real detections), float64 otherwise
    auto mul = [](double p, double q, bool f) { return f ? double(float(p) * float(q)) : p * q; };
    auto dvd = [](double p, double q, bool f) { return f ? double(float(p) / float(q)) : p / q; };
    auto sqr = [](double p, bool f) { return f ? double(sqrtf(float(p))) : sqrt(p); };
    auto sub = [](double p, double q, bool f) { return f ? double(float(p) - float(q)) : p - q; };
    const double w1 = sqr(mul(a.v[2], a.v[3], a.f32), a.f32), h1 = sqr(dvd(a.v[2], a.v[3], a.f32), a.f32);
    const double w2 = sqr(mul(b.v[2], b.v[3], b.f32), b.f32), h2 = sqr(dvd(b.v[2], b.v[3], b.f32), b.f32);
    const bool ff = a.f32 && b.f32;
    const double gap = double(i2 - i1);
    const double dx = sub(b.v[0], a.v[0], ff) / gap, dy = sub(b.v[1], a.v[1], ff) / gap;
    const double dw = sub(w2, w1, ff) / gap, dh = sub(h2, h1, ff) / gap;
    for (int i = 0; i < 7; ++i) x[i] = sx[i];
    for (int i = 0; i < 49; ++i) P[i] = sP[i];
    hist = shist;
    observed = true;
    const int n = i2 - i1;
    for (int i = 0; i < n; ++i) {
      const double w = w1 + (i + 1) * dw, h = h1 + (i + 1) * dh;
      Meas m;
      m.some = true;
      m.f32 = false;
      m.v[0] = a.v[0] + (i + 1) * dx;
      m.v[1] = a.v[1] + (i + 1) * dy;
      m.v[2] = w * h;
      m.v[3] = w / h;
      hist.push(m);
      correct(m.v);
      if (i != n - 1) predict();
    }
  }

  OCS_HD void update(const Meas& z) {      // kalmanfilter.py:107-131, z present
    hist.push(z);
    if (!observed && has_saved) unfreeze();
    observed = true;
    correct(z.v);
  }
};

OCS_HD Meas box_to_z(const float* b) {    // ocsort.py:21-33, float32 arithmetic
  const float w = b[2] - b[0], h = b[3] - b[1];
  Meas m;
  m.some = true;
  m.f32 = true;
  m.v[0] = b[0] + w / 2.f;
  m.v[1] = b[1] + h / 2.f;
  m.v[2] = w * h;
  m.v[3] = w / (h + 1e-6f);
  return m;
}

OCS_HD void state_to_box(const double* x, double out[4]) {   // ocsort.py:36-45
  const double w = sqrt(x[2] * x[3]), h = x[2] / w;
  out[0] = x[0] - w / 2.;
  out[1] = x[1] - h / 2.;
  out[2] = x[0] + w / 2.;
  out[3] = x[1] + h / 2.;
}

OCS_HD double iou(const double* a, const double* b) {   // association.py:3-20
  const double xx1 = dmax(a[0], b[0]), yy1 = dmax(a[1], b[1]);
  const double xx2 = dmin(a[2], b[2]), yy2 = dmin(a[3], b[3]);
  const double w = dmax(0., xx2 - xx1), h = dmax(0., yy2 - yy1), wh = w * h;
  return wh / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - wh);
}

// `last_observation.sum() >= 0` (ocsort.py:113, 281), summed in float32 left to right
OCS_HD bool box_sum_nonneg(const float b[5]) {
  float s = b[0];
  for (int i = 1; i < 5; ++i) s += b[i];
  return s >= 0.f;
}

// Direction and mean speed update of a track that gets detection b, prev = the observation delta_t frames back
// (ocsort.py:48-53, 113-125): float32 up to the per-age increment, then float64.
OCS_HD void velocity_update(const float* prev, const float* b, int age, double vel[2], double avg_vel[2], double* speed) {
  const float cx1 = (prev[0] + prev[2]) / 2.f, cy1 = (prev[1] + prev[3]) / 2.f;
  const float cx2 = (b[0] + b[2]) / 2.f, cy2 = (b[1] + b[3]) / 2.f;
  const float dy = cy2 - cy1, dx = cx2 - cx1;
  const float norm = sqrtf(dy * dy + dx * dx) + 1e-6f;
  vel[0] = dy / norm;
  vel[1] = dx / norm;
  const float a = static_cast<float>(age);
  avg_vel[0] += static_cast<double>(dy / a);
  avg_vel[1] += static_cast<double>(dx / a);
  *speed = fabs(avg_vel[0]) + fabs(avg_vel[1]);
}

// The angle term of the association cost (ocsort.py:216-218 / association.py:60-82) for a track with direction vel whose
// observation delta_t frames back is pb (pb[4] < 0: none) against a detection box d with score s.
OCS_HD void angle_anchor(const double pb[5], double* valid, double* cx2, double* cy2) {
  *valid = pb[4] < 0. ? 0. : 1.;
  *cx2 = (pb[0] + pb[2]) / 2.;
  *cy2 = (pb[1] + pb[3]) / 2.;
}

OCS_HD double angle_term(double valid, double cx2, double cy2, const double vel[2], const double* d, float s, double inertia) {
  const double cx1 = (d[0] + d[2]) / 2., cy1 = (d[1] + d[3]) / 2.;
  double dx = cx1 - cx2, dy = cy1 - cy2;
  const double norm = sqrt(dx * dx + dy * dy) + 1e-6;
  dx /= norm;
  dy /= norm;
  double c = vel[1] * dx + vel[0] * dy;
  c = dmin(1., dmax(-1., c));
  // c == 0 (tracks that have no direction yet) gives acos = pi/2 and an angle term of exactly 0: skip the call
  const double ang = c == 0. ? 0. : (M_PI / 2.0 - fabs(acos(c))) / M_PI;
  return (valid * ang) * inertia * static_cast<double>(s);
}

}  // namespace ocs
