#include "profile.h"

#include <mutex>
#include <vector>

#include "../../include/mipnerf_b200.h"

namespace mipnerf {
namespace {

struct Slot {
  cudaEvent_t start, stop;
  int id;
};
struct State {
  std::mutex mu;
  bool timing = false;
  int64_t launches[kKernCount] = {0};
  std::vector<Slot> pending;
  std::vector<Slot> free_slots;
  double ms[kKernCount] = {0};
  int64_t timed[kKernCount] = {0};
};
State& state() {
  static State s;
  return s;
}
const char* const kNames[kKernCount] = {"coarse_t",  "cast_rays", "ipe",          "pos_enc",      "linear_f32",
                                        "composite", "resample",  "pack_weights", "mlp_level_tc", "mlp_tc",
                                        "generate_rays", "distloss", "ray_prologue",
                                        "render_backward", "dgrad_f32", "wgrad_f32", "adam", "linear_tc", "wgrad_tc",
                                        "image_metrics", "density_tc", "isosurface", "radiance_tc",
                                        "radiance_dirs_tc", "radiance_pairs", "interlevel_loss", "grid_proposal_backward",
                                        "grid_proposal", "grid_tv", "grid_visibility_bricks",
                                        "grid_render_bricks", "grid_render_backward", "grid_render_u8",
                                        "grid_visibility", "grid_render"};

}  // namespace

const char* kernel_name(int id) { return (id >= 0 && id < kKernCount) ? kNames[id] : "?"; }

LaunchScope::LaunchScope(int id, cudaStream_t st) : id_(id), st_(st), slot_(-1) {
  State& s = state();
  std::lock_guard<std::mutex> g(s.mu);
  s.launches[id]++;
  if (!s.timing) return;
  Slot sl;
  if (!s.free_slots.empty()) {
    sl = s.free_slots.back();
    s.free_slots.pop_back();
  } else {
    if (cudaEventCreate(&sl.start) != cudaSuccess || cudaEventCreate(&sl.stop) != cudaSuccess) return;
  }
  sl.id = id;
  cudaEventRecord(sl.start, st);
  s.pending.push_back(sl);
  slot_ = (int)s.pending.size() - 1;
}

LaunchScope::~LaunchScope() {
  if (slot_ < 0) return;
  State& s = state();
  std::lock_guard<std::mutex> g(s.mu);
  if (slot_ < (int)s.pending.size()) cudaEventRecord(s.pending[slot_].stop, st_);
}

}  // namespace mipnerf

extern "C" {

int mipnerf_b200_profile_enable(int timing_on) {
  mipnerf::State& s = mipnerf::state();
  std::lock_guard<std::mutex> g(s.mu);
  s.timing = timing_on != 0;
  return MIPNERF_B200_OK;
}

int mipnerf_b200_profile_num_kernels(void) { return mipnerf::kKernCount; }

const char* mipnerf_b200_profile_kernel_name(int kernel_id) { return mipnerf::kernel_name(kernel_id); }

int mipnerf_b200_profile_read(int kernel_id, int64_t* launches, double* timed_ms, int64_t* timed_launches,
                              int reset) {
  if (kernel_id < 0 || kernel_id >= mipnerf::kKernCount) return MIPNERF_B200_EINVAL;
  mipnerf::State& s = mipnerf::state();
  std::lock_guard<std::mutex> g(s.mu);
  // fold finished event pairs (synchronises on each pending stop event)
  for (auto& sl : s.pending) {
    float ms = 0.f;
    if (cudaEventSynchronize(sl.stop) == cudaSuccess && cudaEventElapsedTime(&ms, sl.start, sl.stop) == cudaSuccess) {
      s.ms[sl.id] += ms;
      s.timed[sl.id]++;
    }
    s.free_slots.push_back(sl);
  }
  s.pending.clear();
  if (launches) *launches = s.launches[kernel_id];
  if (timed_ms) *timed_ms = s.ms[kernel_id];
  if (timed_launches) *timed_launches = s.timed[kernel_id];
  if (reset) {
    s.launches[kernel_id] = 0;
    s.ms[kernel_id] = 0;
    s.timed[kernel_id] = 0;
  }
  return MIPNERF_B200_OK;
}

}  // extern "C"
