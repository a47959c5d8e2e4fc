// esvo_b200 -- the closed ESVO loop on one event stream: time surfaces, SGM start-up, mapping and tracking as one system.
//
// The reference runs four ROS nodes (two esvo_time_surface, esvo_Mapping, esvo_Tracking) that talk through topics, tf and
// the /ESVO_SYSTEM_STATUS parameter.  esvo_System owns one CameraSystem (one esvo_ctx), both TimeSurfaces, the mapper,
// the tracker and the tf pose buffer both nodes look poses up in, and runs the nodes on a fixed schedule of sync ticks
// t_k = t0 + k * dt (DESIGN.md section 5):
//   1. every event with stamp < t_k that has not been delivered goes to both time surfaces; the mapper and the tracker read
//      their left events from camera 0's time-surface log (esvo_events_window_dev, esvo_events_lower_bound_dev) and only
//      learn how many there are -- their host event buffers stay empty;
//   2. both time surfaces are built at t_k; the pair goes to the mapper's history, the left image to the tracker's -- on the
//      device: the mapper's history is the context's time-surface history, the tracker reads the newest camera-0 build;
//   3. esvo_Tracking::TrackingLoopOnce(); a pose it produces goes into the pose buffer at once (publishPose ->
//      stampedPoseCallback);
//   4. every mapping_every-th tick esvo_Mapping::MappingLoopOnce(); a map it publishes goes to the tracker's
//      refMapCallback with the map's stamp -- published and adopted on the device (esvo_map_publish_dev,
//      esvo_track_adopt_map_dev), never downloaded.
// Where a reference node calls exit(-1) the system sets the status to TERMINATE, keeps the reason in error_ and stops.
// Header-only; link with libesvo_b200.so.
#pragma once
#include <chrono>

#include "esvo_core.hpp"

// esvo::PoseBuffer, the tf pose buffer both nodes look poses up in, lives in esvo_core.hpp (the MVStereo node owns one too).

namespace esvo_core {

class esvo_System {
 public:
  struct Config {
    int64_t t0_ns = 0, dt_ns = 10000000;   // sync ticks; 100 Hz as stereo_time_surface.launch (system_hkust.launch: 50 Hz)
    int mapping_every = 5;                 // round(mapping period / dt): mapping_rate_hz 20 at 100 Hz ticks
    // cfg/mapping/mapping_hkust.yaml
    size_t PROCESS_EVENT_NUM = 1000, TS_HISTORY_LENGTH = 100, INIT_SGM_DP_NUM_THRESHOLD = 500;
    double BM_half_slice_thickness = 0.001;
    bool Denoising = true;
    // cfg/tracking/tracking_hkust.yaml
    size_t TRK_TS_HISTORY_LENGTH = 100, REF_HISTORY_LENGTH = 10;
    core::RegProblemType rpType = core::REG_ANALYTICAL;
  };
  struct TickRecord { int64_t t = 0; std::string status; bool has_pose = false; esvo::Pose T{}; double ts_ms = 0, tracking_ms = 0, mapping_ms = 0; };
  struct MappingRecord {
    size_t tick = 0; int ran = 0; bool ok = false; size_t n_sgm_points = 0; esvo_Mapping::Counters ctr{};
    bool published = false; size_t cloud_points = 0; int64_t stamp = 0;
  };

  esvo_System(esvo::CameraSystem::Ptr cs, const Config& cfg)
      : cfg_(cfg), cs_(cs), ts_left_(cs, 0), ts_right_(cs, 1), mapper_(cs), tracker_(cs, cfg.rpType, cfg.TRK_TS_HISTORY_LENGTH, cfg.REF_HISTORY_LENGTH) {
    mapper_.PROCESS_EVENT_NUM_ = cfg.PROCESS_EVENT_NUM; mapper_.TS_HISTORY_LENGTH_ = cfg.TS_HISTORY_LENGTH;
    mapper_.INIT_SGM_DP_NUM_Threshold_ = cfg.INIT_SGM_DP_NUM_THRESHOLD; mapper_.BM_half_slice_thickness_ = cfg.BM_half_slice_thickness;
    mapper_.bDenoising_ = cfg.Denoising;
    auto poseAt = [this](int64_t t, esvo::Pose& T) { return poses_.lookup(t, T); };
    mapper_.setPoseProvider(poseAt);
    tracker_.setPoseProvider(poseAt);
    esvo_track_srand(cs->ctx(), 1);        // the reference never seeds rand(): glibc seed 1
    if (esvo_ts_history_reserve_dev(cs->ctx(), cfg.TS_HISTORY_LENGTH) != ESVO_OK)
      throw std::runtime_error(std::string("esvo_ts_history_reserve_dev: ") + esvo_last_error(cs->ctx()));
  }
  int64_t nextTick() const { return cfg_.t0_ns + (int64_t)k_ * cfg_.dt_ns; }
  // One sync tick.  left / right: the events with stamp < nextTick() not delivered yet, time-ordered.  false once stopped.
  bool SpinOnce(const std::vector<esvo::Event>& left, const std::vector<esvo::Event>& right) {
    return spin([&] { return (left.empty() || ts_left_.eventsCallback(left)) && (right.empty() || ts_right_.eventsCallback(right)); });
  }
  // The same tick with the events as packed runs of wire records (e.g. EventArray messages of a ROS bag,
  // esvo::RosBagEvents::takeBefore): same schedule, records and outputs as the vector form on the same events.
  bool SpinOnce(const std::vector<esvo::EventRun>& left, const std::vector<esvo::EventRun>& right) {
    return spin([&] { return ts_left_.eventsCallback(left) && ts_right_.eventsCallback(right); });
  }
  // the fused map the mapper holds (DepthMap element order)
  void getMap(std::vector<esvo::DepthPoint>& out) { core::DepthFusion f(cs_); f.getElements(out); }
  bool saveTrajectory(const std::string& path) const { return tracker_.saveTrajectory(path); }
  // host time of each call SpinOnce makes, and of each call MappingLoopOnce makes (names "mapping.*" inside it)
  esvo::CallTimes callTimes() const {
    esvo::CallTimes all = calls_;
    for (const auto& e : mapper_.calls_.ms) all.ms[e.first] = e.second;
    return all;
  }

  const Config& config() const { return cfg_; }
  std::string status_ = "INITIALIZATION";   // /ESVO_SYSTEM_STATUS
  std::string error_;
  std::vector<TickRecord> ticks_;
  std::vector<MappingRecord> mapping_;
  esvo::PoseBuffer poses_;

 private:
  // one sync tick; push() hands the tick's events to both time surfaces
  template <class Push>
  bool spin(Push&& push) {
    if (status_ == "TERMINATE") return false;
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    TickRecord rec;
    rec.t = nextTick();
    const auto c0 = clk::now();
    bool ok;
    { auto _ = calls_.time("ts.eventsCallback"); ok = push(); }
    // the mapper and the tracker read their left events from camera 0's log (esvo_events_*_dev): they get the count only
    { auto _ = calls_.time("mapping.eventsCallback"); mapper_.eventsCallback(ts_left_.eventsPushed()); }
    { auto _ = calls_.time("tracking.eventsCallback"); tracker_.eventsCallback(ts_left_.eventsPushed()); }
    { auto _ = calls_.time("ts.createTimeSurfaceAtTime");
      ok = ok && ts_left_.createTimeSurfaceAtTime(rec.t, nullptr) && ts_right_.createTimeSurfaceAtTime(rec.t, nullptr); }
    if (!ok) return stop(std::string("time surface: ") + esvo_last_error(cs_->ctx()), rec);
    { auto _ = calls_.time("mapping.timeSurfaceCallback");
      if (!mapper_.timeSurfaceCallback(rec.t)) return stop(std::string("time-surface history: ") + esvo_last_error(cs_->ctx()), rec); }
    { auto _ = calls_.time("tracking.timeSurfaceCallback"); tracker_.timeSurfaceCallback(rec.t); }
    const auto c1 = clk::now();
    tracker_.ESVO_System_Status_ = status_;
    { auto _ = calls_.time("tracking.TrackingLoopOnce"); rec.has_pose = tracker_.TrackingLoopOnce(); }
    status_ = tracker_.ESVO_System_Status_;
    if (!tracker_.error_.empty()) return stop("tracking: " + tracker_.error_, rec);
    if (rec.has_pose) { rec.T = tracker_.T_world_cur_; poses_.setTransform(tracker_.cur_.t_, tracker_.cur_.tr_); }
    const auto c2 = clk::now();
    if (k_ % (size_t)cfg_.mapping_every == 0) {
      mapper_.ESVO_System_Status_ = status_;
      esvo_Mapping::LoopResult r;
      { auto _ = calls_.time("mapping.MappingLoopOnce"); mapper_.MappingLoopOnce(r); }
      if (!mapper_.error_.empty()) return stop("mapping: " + mapper_.error_, rec);
      status_ = mapper_.ESVO_System_Status_;
      MappingRecord m;
      m.tick = k_; m.ran = r.ran; m.ok = r.ok; m.n_sgm_points = r.n_sgm_points; m.ctr = r.ctr;
      m.published = r.published; m.cloud_points = r.cloud_points; m.stamp = r.stamp;
      if (r.published) tracker_.refMapCallback(r.stamp, r.cloud_points);
      mapping_.push_back(m);
    }
    const auto c3 = clk::now();
    rec.ts_ms = ms(c0, c1); rec.tracking_ms = ms(c1, c2); rec.mapping_ms = ms(c2, c3);
    rec.status = status_;
    ticks_.push_back(rec);
    ++k_;
    return true;
  }
  bool stop(const std::string& why, TickRecord& rec) {
    error_ = why; status_ = "TERMINATE";
    rec.status = status_; ticks_.push_back(rec); ++k_;
    return false;
  }
  Config cfg_;
  esvo::CameraSystem::Ptr cs_;
  esvo_time_surface::TimeSurface ts_left_, ts_right_;
  esvo_Mapping mapper_;
  esvo_Tracking tracker_;
  esvo::CallTimes calls_;
  size_t k_ = 0;
};

}  // namespace esvo_core
