// esvo_b200 -- the multi-view stereo system on one event stream with known poses: time surfaces and the esvo_MVStereo node
// as one loop (launch/mvstereo/mvstereo_{rpg,upenn}.launch).
//
// The reference runs three ROS nodes (two esvo_time_surface, esvo_MVStereo) fed by a recorded stream whose ground-truth
// poses arrive on the stamped_pose topic.  esvo_MVStereoSystem owns one CameraSystem (one esvo_ctx), both TimeSurfaces and
// the node (with its tf pose buffer), and runs them on a fixed schedule of sync ticks t_k = t0 + k * dt (DESIGN.md
// section 5):
//   1. every event with stamp < t_k that has not been delivered goes to both time surfaces and to the node's left / right
//      queues (eventsCallback);
//   2. both time surfaces are built at t_k and the pair goes to the node's history (timeSurfaceCallback);
//   3. every mapping_every-th tick (mapping_every = round(1 / (mapping_rate_hz * dt))): every pose with stamp <= t_k not
//      delivered yet goes to stampedPoseCallback in stream order, then one pass of MappingLoop (MappingLoopOnce).
// Header-only; link with libesvo_b200.so.
#pragma once
#include <chrono>
#include <cmath>

#include "esvo_core.hpp"

namespace esvo_core {

class esvo_MVStereoSystem {
 public:
  // cfg/mvstereo/mvstereo_{rpg,upenn}.yaml keys the loop reads (the rest travel in esvo_params); defaults = the node's
  // constructor defaults (esvo_MVStereo.cpp:71-101)
  struct Config {
    int64_t t0_ns = 0, dt_ns = 20000000;   // sync ticks; 50 Hz as mvstereo_{rpg,upenn}.launch (rostopic pub -r 50 /sync)
    double mapping_rate_hz = 20;
    int MVStereoMode = 1;
    size_t PROCESS_EVENT_NUM = 500, TS_HISTORY_LENGTH = 100, EM_NUM_EVENT_MATCHING = 3000;
    double BM_half_slice_thickness = 0.001;
    double EM_Slice_Thickness = 1e-3, EM_Time_THRESHOLD = 5e-5, EM_EPIPOLAR_THRESHOLD = 0.5, EM_TS_NCC_THRESHOLD = 0.1;
    bool Denoising = false;
    bool marker_frame = false;             // dvs_frame_id "marker" (the rpg launch): poses are the marker's
    int mappingEvery() const { return std::max(1, (int)std::lround(1e9 / (mapping_rate_hz * (double)dt_ns))); }
  };
  struct FrameRecord {
    size_t tick = 0; int64_t t = 0; size_t resets = 0;   // resets: of the node so far
    esvo_MVStereo::LoopResult r;           // cloud emptied; its size is kept in cloud_points
    size_t cloud_points = 0;
    double ms = 0;
  };

  esvo_MVStereoSystem(esvo::CameraSystem::Ptr cs, const Config& cfg)
      : cfg_(cfg), cs_(cs), ts_left_(cs, 0), ts_right_(cs, 1), node_(cs, (esvo_MVStereo::eMVStereoMode)cfg.MVStereoMode),
        img_l_((size_t)cs->width_ * cs->height_), img_r_((size_t)cs->width_ * cs->height_) {
    MVStereoFrontEnd& n = node_.node_;
    n.PROCESS_EVENT_NUM_ = cfg.PROCESS_EVENT_NUM; n.TS_HISTORY_LENGTH_ = cfg.TS_HISTORY_LENGTH;
    n.EM_numEventMatching_ = cfg.EM_NUM_EVENT_MATCHING; n.BM_half_slice_thickness_ = cfg.BM_half_slice_thickness;
    n.bDenoising_ = cfg.Denoising; n.marker_frame_ = cfg.marker_frame;
    node_.resetEMParameters(cfg.EM_Slice_Thickness, cfg.EM_Time_THRESHOLD, cfg.EM_EPIPOLAR_THRESHOLD, cfg.EM_TS_NCC_THRESHOLD);
    node_.setPoseProvider([this](int64_t t, esvo::Pose& T) { return node_.getPoseAt(t, T); });
  }
  int64_t nextTick() const { return cfg_.t0_ns + (int64_t)k_ * cfg_.dt_ns; }
  bool isMappingTick() const { return k_ % (size_t)cfg_.mappingEvery() == 0; }
  // One sync tick.  left / right: the events with stamp < nextTick() not delivered yet, time-ordered; poses: (stamp,
  // T_world_dvs) with stamp <= nextTick() not delivered yet, consumed only on a mapping tick (isMappingTick()).  false
  // (and error_ set) when a time-surface call fails or the device reports an error after a mapping pass; an ABI call
  // refused inside MappingAtTime is not told apart from an empty result.
  bool SpinOnce(const std::vector<esvo::Event>& left, const std::vector<esvo::Event>& right,
                const std::vector<std::pair<int64_t, esvo::Pose>>& poses) {
    if (!error_.empty()) return false;
    const int64_t t = nextTick();
    const bool ok = (left.empty() || ts_left_.eventsCallback(left)) && (right.empty() || ts_right_.eventsCallback(right)) &&
                    ts_left_.createTimeSurfaceAtTime(t, img_l_.data()) && ts_right_.createTimeSurfaceAtTime(t, img_r_.data());
    if (!ok) { error_ = std::string("time surface: ") + esvo_last_error(cs_->ctx()); return false; }
    node_.eventsCallback(left, true); node_.eventsCallback(right, false);
    node_.timeSurfaceCallback(t, img_l_.data(), img_r_.data());
    if (isMappingTick()) {
      using clk = std::chrono::steady_clock;
      const auto c0 = clk::now();
      for (const auto& p : poses) node_.stampedPoseCallback(p.first, p.second);
      FrameRecord f;
      f.tick = k_; f.t = t;
      node_.MappingLoopOnce(f.r);
      f.resets = node_.node_.n_resets_;
      f.cloud_points = f.r.cloud.size() / 3;
      std::vector<float>().swap(f.r.cloud);
      // A CUDA fault inside the pass surfaces here; MappingAtTime reports only "no result" (ok = false), like the reference.
      const bool device_ok = esvo_sync(cs_->ctx()) == ESVO_OK;
      f.ms = std::chrono::duration<double, std::milli>(clk::now() - c0).count();
      frames_.push_back(std::move(f));
      if (!device_ok) { error_ = std::string("mapping: ") + esvo_last_error(cs_->ctx()); ++k_; return false; }
    }
    ++k_;
    return true;
  }
  // the map of the node's current DepthFrame (DepthMap element order)
  void getMap(std::vector<esvo::DepthPoint>& out) { node_.getMap(out); }
  esvo_MVStereo& node() { return node_; }
  const Config& config() const { return cfg_; }
  std::string error_;
  std::vector<FrameRecord> frames_;

 private:
  Config cfg_;
  esvo::CameraSystem::Ptr cs_;
  esvo_time_surface::TimeSurface ts_left_, ts_right_;
  esvo_MVStereo node_;
  std::vector<uint8_t> img_l_, img_r_;
  size_t k_ = 0;
};

}  // namespace esvo_core
