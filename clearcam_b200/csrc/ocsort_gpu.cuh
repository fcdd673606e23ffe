// The device tracker's handle and slot records, shared by ocsort_gpu.cu (the tracker) and events_gpu.cu (the object
// events that read a slot's live track ids after each step).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace ocsg {

constexpr int kLaneId = 11;          // 4-byte lane holding each track's id (ocsort_gpu.cu I_ID), ascending in slot order

struct SlotCfg {
  double* dl;
  int32_t* il;
  int cap, active;
  int max_age, min_hits, delta_t, use_byte;
  double iou_threshold, inertia;
};
struct SlotCnt { int T, frame_count, next_id, pad; };

}  // namespace ocsg

struct cc_events;                    // events_gpu.cu: per-slot event configuration and state
struct cc_alerts;                    // alerts_gpu.cu: per-slot alert configuration and state

struct cc_ocsort_gpu {
  int S = 0, rb = 0;                 // slots; ring entries per track (max delta_t + 2)
  std::vector<ocsg::SlotCfg> cfg;    // host copy of every slot's configuration
  ocsg::SlotCfg* d_cfg = nullptr;
  ocsg::SlotCnt* d_cnt = nullptr;
  cc_events* ev = nullptr;           // made by the first cc_ocsort_gpu_events_configure
  cc_alerts* al = nullptr;           // made by the first cc_ocsort_gpu_alerts_configure
};

// events_gpu.cu: a slot's event state follows its tracker (configure clears it, free frees it); destroy frees all
int cc_events_slot_clear(cc_ocsort_gpu* h, int slot, cudaStream_t st);
int cc_events_slot_free(cc_ocsort_gpu* h, int slot, cudaStream_t st);
void cc_events_destroy(cc_ocsort_gpu* h);

// alerts_gpu.cu: a slot's alerts follow its tracker too (configure clears the object counter and the warm-up, free frees
// them); destroy frees all
int cc_alerts_slot_clear(cc_ocsort_gpu* h, int slot, cudaStream_t st);
int cc_alerts_slot_free(cc_ocsort_gpu* h, int slot, cudaStream_t st);
void cc_alerts_destroy(cc_ocsort_gpu* h);
