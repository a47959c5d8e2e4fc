// esvo_b200 -- the closed ESVO loop on one event stream: time surfaces, SGM start-up, mapping and tracking as one system.
//
// The reference runs four ROS nodes (two esvo_time_surface, esvo_Mapping, esvo_Tracking) that talk through topics, tf and
// the /ESVO_SYSTEM_STATUS parameter.  esvo_System owns one CameraSystem (one esvo_ctx), both TimeSurfaces, the mapper,
// the tracker and the tf pose buffer both nodes look poses up in, and runs the nodes on a fixed schedule of sync ticks
// t_k = t0 + k * dt (DESIGN.md section 5):
//   1. every event with stamp < t_k that has not been delivered goes to both time surfaces, the mapper's left / right
//      buffers and the tracker's left buffer;
//   2. both time surfaces are built at t_k; the pair goes to the mapper's history, the left image to the tracker's;
//   3. esvo_Tracking::TrackingLoopOnce(); a pose it produces goes into the pose buffer at once (publishPose ->
//      stampedPoseCallback);
//   4. every mapping_every-th tick esvo_Mapping::MappingLoopOnce(); a map it publishes goes to the tracker's
//      refMapCallback with the map's stamp.
// Where a reference node calls exit(-1) the system sets the status to TERMINATE, keeps the reason in error_ and stops.
// Header-only; link with libesvo_b200.so.
#pragma once
#include <chrono>

#include "esvo_core.hpp"

namespace esvo {

// The tf::Transformer(true, ros::Duration(100.0)) both nodes keep (esvo_Mapping.cpp:140, esvo_Tracking.cpp:58), filled by
// stampedPoseCallback and read by getPoseAt.  Restates the tf2 TimeCache behaviour the nodes rely on (DESIGN.md section 2):
//  * the pose travels as quaternion + position (PoseStamped) and comes back as a 4x4: q = Eigen::Quaterniond(R) on the way
//    in, R = q.toRotationMatrix() on the way out -- an exact stamp returns the stored pose after that round trip;
//  * between two stamps: translation (1 - r) p0 + r p1, rotation tf2 slerp (shortest path), r = (t - t0) / (t1 - t0) in
//    seconds of ros::Duration;
//  * no extrapolation: before the oldest or after the newest stamp there is no pose; one entry answers only at its stamp;
//    stamp 0 means "the latest";
//  * entries older than the newest minus the cache time (100 s) are dropped; a second pose for a stored stamp is refused.
class PoseBuffer {
 public:
  explicit PoseBuffer(int64_t cache_ns = 100000000000LL) : cache_ns_(cache_ns) {}
  bool setTransform(int64_t stamp_ns, const Pose& T_world_dvs) {
    if (!s_.empty() && s_.back().t > stamp_ns + cache_ns_) return false;
    auto it = std::lower_bound(s_.begin(), s_.end(), stamp_ns, [](const Entry& e, int64_t t) { return e.t < t; });
    if (it != s_.end() && it->t == stamp_ns) return false;
    Entry e;
    e.t = stamp_ns;
    const double R[9] = {T_world_dvs[0], T_world_dvs[1], T_world_dvs[2], T_world_dvs[4], T_world_dvs[5], T_world_dvs[6],
                         T_world_dvs[8], T_world_dvs[9], T_world_dvs[10]};
    quaternionFromRotation(R, e.q);
    e.p[0] = T_world_dvs[3]; e.p[1] = T_world_dvs[7]; e.p[2] = T_world_dvs[11];
    s_.insert(it, e);
    while (s_.front().t + cache_ns_ < s_.back().t) s_.erase(s_.begin());
    return true;
  }
  bool canTransform(int64_t t_ns) const { Pose T; return lookup(t_ns, T); }
  bool lookup(int64_t t_ns, Pose& T) const {
    if (s_.empty()) return false;
    if (t_ns == 0) return toPose(s_.back().q, s_.back().p, T);
    if (t_ns < s_.front().t || t_ns > s_.back().t) return false;
    auto it = std::upper_bound(s_.begin(), s_.end(), t_ns, [](int64_t t, const Entry& e) { return t < e.t; });
    const Entry& a = *(it - 1);
    if (a.t == t_ns) return toPose(a.q, a.p, T);
    const Entry& b = *it;
    const double r = esvo_core::frontend::toSec(t_ns - a.t) / esvo_core::frontend::toSec(b.t - a.t);   // ros::Duration::toSec()
    double q[4], p[3];
    for (int i = 0; i < 3; ++i) p[i] = (1.0 - r) * a.p[i] + r * b.p[i];
    slerp(a.q, b.q, r, q);
    return toPose(q, p, T);
  }
  size_t size() const { return s_.size(); }
  void clear() { s_.clear(); }
  // tf2::Quaternion::slerp / angleShortestPath (tf2Acos clamps to [-1, 1]); q = x, y, z, w
  static void slerp(const double a[4], const double b[4], double t, double out[4]) {
    auto dot = [](const double* u, const double* v) { return u[0] * v[0] + u[1] * v[1] + u[2] * v[2] + u[3] * v[3]; };
    const double s = std::sqrt(dot(a, a) * dot(b, b)), d_ab = dot(a, b);
    const double c = std::max(-1.0, std::min(1.0, (d_ab < 0 ? -d_ab : d_ab) / s));
    const double theta = std::acos(c) * 2.0 / 2.0;
    if (theta == 0.0) { std::copy(a, a + 4, out); return; }
    const double d = 1.0 / std::sin(theta), s0 = std::sin((1.0 - t) * theta), s1 = std::sin(t * theta);
    const double sg = d_ab < 0 ? -1.0 : 1.0;
    for (int i = 0; i < 4; ++i) out[i] = (a[i] * s0 + sg * b[i] * s1) * d;
  }
 private:
  struct Entry { int64_t t; double q[4]; double p[3]; };
  static bool toPose(const double q[4], const double p[3], Pose& T) {
    double R[9];
    rotationFromQuaternion(q, R);
    T = {R[0], R[1], R[2], p[0], R[3], R[4], R[5], p[1], R[6], R[7], R[8], p[2], 0, 0, 0, 1};
    return true;
  }
  int64_t cache_ns_;
  std::vector<Entry> s_;   // oldest first
};

}  // namespace esvo

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
      : cfg_(cfg), cs_(cs), ts_left_(cs, 0), ts_right_(cs, 1), mapper_(cs), tracker_(cs, cfg.rpType, cfg.TRK_TS_HISTORY_LENGTH, cfg.REF_HISTORY_LENGTH),
        img_l_((size_t)cs->width_ * cs->height_), img_r_((size_t)cs->width_ * cs->height_) {
    mapper_.PROCESS_EVENT_NUM_ = cfg.PROCESS_EVENT_NUM; mapper_.TS_HISTORY_LENGTH_ = cfg.TS_HISTORY_LENGTH;
    mapper_.INIT_SGM_DP_NUM_Threshold_ = cfg.INIT_SGM_DP_NUM_THRESHOLD; mapper_.BM_half_slice_thickness_ = cfg.BM_half_slice_thickness;
    mapper_.bDenoising_ = cfg.Denoising;
    auto poseAt = [this](int64_t t, esvo::Pose& T) { return poses_.lookup(t, T); };
    mapper_.setPoseProvider(poseAt);
    tracker_.setPoseProvider(poseAt);
    esvo_track_srand(cs->ctx(), 1);        // the reference never seeds rand(): glibc seed 1
  }
  int64_t nextTick() const { return cfg_.t0_ns + (int64_t)k_ * cfg_.dt_ns; }
  // One sync tick.  left / right: the events with stamp < nextTick() not delivered yet, time-ordered.  false once stopped.
  bool SpinOnce(const std::vector<esvo::Event>& left, const std::vector<esvo::Event>& right) {
    if (status_ == "TERMINATE") return false;
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    TickRecord rec;
    rec.t = nextTick();
    const auto c0 = clk::now();
    bool ok = (left.empty() || ts_left_.eventsCallback(left)) && (right.empty() || ts_right_.eventsCallback(right));
    mapper_.eventsCallback(left, true); mapper_.eventsCallback(right, false);
    tracker_.eventsCallback(left);
    ok = ok && ts_left_.createTimeSurfaceAtTime(rec.t, img_l_.data()) && ts_right_.createTimeSurfaceAtTime(rec.t, img_r_.data());
    if (!ok) return stop(std::string("time surface: ") + esvo_last_error(cs_->ctx()), rec);
    mapper_.timeSurfaceCallback(rec.t, img_l_.data(), img_r_.data());
    tracker_.timeSurfaceCallback(rec.t, img_l_.data());
    const auto c1 = clk::now();
    tracker_.ESVO_System_Status_ = status_;
    rec.has_pose = tracker_.TrackingLoopOnce();
    status_ = tracker_.ESVO_System_Status_;
    if (!tracker_.error_.empty()) return stop("tracking: " + tracker_.error_, rec);
    if (rec.has_pose) { rec.T = tracker_.T_world_cur_; poses_.setTransform(tracker_.cur_.t_, tracker_.cur_.tr_); }
    const auto c2 = clk::now();
    if (k_ % (size_t)cfg_.mapping_every == 0) {
      mapper_.ESVO_System_Status_ = status_;
      esvo_Mapping::LoopResult r;
      mapper_.MappingLoopOnce(r);
      status_ = mapper_.ESVO_System_Status_;
      MappingRecord m;
      m.tick = k_; m.ran = r.ran; m.ok = r.ok; m.n_sgm_points = r.n_sgm_points; m.ctr = r.ctr;
      m.published = r.published; m.cloud_points = r.cloud.size() / 3; m.stamp = r.stamp;
      if (r.published) tracker_.refMapCallback(r.stamp, r.cloud);
      mapping_.push_back(m);
    }
    const auto c3 = clk::now();
    rec.ts_ms = ms(c0, c1); rec.tracking_ms = ms(c1, c2); rec.mapping_ms = ms(c2, c3);
    rec.status = status_;
    ticks_.push_back(rec);
    ++k_;
    return true;
  }
  // the fused map the mapper holds (DepthMap element order)
  void getMap(std::vector<esvo::DepthPoint>& out) { core::DepthFusion f(cs_); f.getElements(out); }
  bool saveTrajectory(const std::string& path) const { return tracker_.saveTrajectory(path); }

  const Config& config() const { return cfg_; }
  std::string status_ = "INITIALIZATION";   // /ESVO_SYSTEM_STATUS
  std::string error_;
  std::vector<TickRecord> ticks_;
  std::vector<MappingRecord> mapping_;
  esvo::PoseBuffer poses_;

 private:
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
  std::vector<uint8_t> img_l_, img_r_;
  size_t k_ = 0;
};

}  // namespace esvo_core
