// esvo_b200 -- C++ host shim over the C ABI (include/esvo_b200.h).
//
// ROS-free mirror of the reference's class surface for the hot path, so that code written against
// esvo_core::core::{EventBM, DepthProblemSolver, DepthFusion, RegProblemSolverLM} and
// esvo_time_surface::TimeSurface keeps its shape: same class and method names, same argument meaning,
// same "bool return for data-dependent failure, no exceptions" convention
// (reference: esvo_core/include/esvo_core/core/*.h, esvo_time_surface/include/esvo_time_surface/TimeSurface.h).
// ROS / Eigen / OpenCV types are replaced by plain structs: ros::Time -> int64 ns, Transformation -> row-major
// double[16], cv::Mat mono8 -> uint8_t*, dvs_msgs::Event -> esvo::Event.  Header-only; link with libesvo_b200.so.
#pragma once
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../esvo_b200.h"

namespace esvo {

struct Event { uint16_t x, y; int64_t ts; bool polarity; };            // dvs_msgs::Event
// n dvs_msgs::Event wire records (13 bytes each, as serialised in a ROS bag) at data; see esvo_ts_push_event_array
struct EventRun { const uint8_t* data = nullptr; size_t n = 0; };
using Pose = std::array<double, 16>;                                    // Transformation (T_world_cam, row-major)
using StampTransformationMap = std::vector<std::pair<int64_t, Pose>>;   // sorted by stamp
using EventMatchPair = esvo_seed;                                       // core::EventMatchPair
using DepthPoint = esvo_depth_point;                                    // container::DepthPoint

namespace detail {
// a StampTransformationMap as the ABI takes it: stamps[n] and row-major poses[16 n]
inline std::pair<std::vector<int64_t>, std::vector<double>> stampsAndPoses(const StampTransformationMap& st_map) {
  std::pair<std::vector<int64_t>, std::vector<double>> sp;
  for (auto& st : st_map) { sp.first.push_back(st.first); sp.second.insert(sp.second.end(), st.second.begin(), st.second.end()); }
  return sp;
}
}  // namespace detail

// container::CameraSystem + the parameter yaml of one node: owns the esvo_ctx of one event stream / GPU.
class CameraSystem {
 public:
  using Ptr = std::shared_ptr<CameraSystem>;
  CameraSystem(const esvo_calib& left, const esvo_calib& right, const esvo_params& params, int device = 0) {
    int st = 0;
    ctx_ = esvo_create(device, &left, &right, &params, &st);
    if (!ctx_) throw std::runtime_error("esvo_create failed with status " + std::to_string(st) + " (no CPU fallback)");
    params_ = params; width_ = left.width; height_ = left.height;
    std::copy(left.P, left.P + 12, P_left_);
    double d[4]; esvo_get_derived(ctx_, d); baseline_ = d[0];
  }
  ~CameraSystem() { esvo_destroy(ctx_); }
  CameraSystem(const CameraSystem&) = delete;
  CameraSystem& operator=(const CameraSystem&) = delete;
  esvo_ctx* ctx() const { return ctx_; }
  const esvo_params& params() const { return params_; }
  int width_ = 0, height_ = 0;
  double baseline_ = 0;
  double P_left_[12] = {0};   // cam_left_ptr_->P_
 private:
  esvo_ctx* ctx_ = nullptr;
  esvo_params params_;
};

// container::TimeSurfaceObservation (stereo mono8 pair + pose); images are borrowed, not copied.
struct TimeSurfaceObservation {
  const uint8_t* left = nullptr;    // nullptr = "the image esvo_ts_build produced on the device"
  const uint8_t* right = nullptr;
  Pose tr_{};
  size_t id_ = 0;
  bool stored_ = false;             // the pair the device history holds under this observation's stamp (esvo_ts_history_store_dev)
  void setTransformation(const Pose& tr) { tr_ = tr; }
};
using StampedTimeSurfaceObs = std::pair<int64_t, TimeSurfaceObservation>;

// Host time and call count per named call, accumulated over a run (scripts/loop_probe.py reports them).
struct CallTimes {
  struct Scope {
    CallTimes* c; const char* name; std::chrono::steady_clock::time_point t0;
    ~Scope() {
      auto& e = c->ms[name];
      e.first += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      ++e.second;
    }
  };
  Scope time(const char* name) { return Scope{this, name, std::chrono::steady_clock::now()}; }
  std::map<std::string, std::pair<double, size_t>> ms;   // name -> (total ms, calls)
};

// Eigen::Quaterniond(const Matrix3d&) (Eigen/src/Geometry/Quaternion.h, quaternion_assign_impl): R row-major 3x3, q = x, y, z, w
inline void quaternionFromRotation(const double R[9], double q[4]) {
  auto m = [&](int r, int c) { return R[3 * r + c]; };
  double t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0) {
    t = std::sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m(2, 1) - m(1, 2)) * t; q[1] = (m(0, 2) - m(2, 0)) * t; q[2] = (m(1, 0) - m(0, 1)) * t;
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m(k, j) - m(j, k)) * t; q[j] = (m(j, i) + m(i, j)) * t; q[k] = (m(k, i) + m(i, k)) * t;
  }
}
// QuaternionBase::toRotationMatrix (same file): q = x, y, z, w -> R row-major 3x3 (no normalisation)
inline void rotationFromQuaternion(const double q[4], double R[9]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}

}  // namespace esvo

namespace esvo_time_surface {
// esvo_time_surface::TimeSurface (TimeSurface.h:98-170) without the ROS node handle: the three callbacks
// become plain methods, the published image is returned to the caller.
class TimeSurface {
 public:
  TimeSurface(esvo::CameraSystem::Ptr cs, int cam) : cs_(std::move(cs)), cam_(cam) {}
  // eventsCallback (TimeSurface.cpp:403-425)
  bool eventsCallback(const std::vector<esvo::Event>& events) {
    x_.resize(events.size()); y_.resize(events.size()); t_.resize(events.size()); p_.resize(events.size());
    for (size_t i = 0; i < events.size(); ++i) { x_[i] = events[i].x; y_[i] = events[i].y; t_[i] = events[i].ts; p_[i] = events[i].polarity; }
    return esvo_ts_push_events(cs_->ctx(), cam_, x_.data(), y_.data(), t_.data(), p_.data(), events.size()) == ESVO_OK;
  }
  // The same on packed runs of wire records (the events of one or more EventArray messages): copied as they are and
  // decoded on the device (esvo_ts_push_event_array), no per-event host work.  With a hot-pixel mask installed
  // (esvo_hotpix_select) the events at hot pixels are dropped.
  bool eventsCallback(const std::vector<esvo::EventRun>& runs) {
    run_ptr_.clear(); run_n_.clear();
    for (const auto& r : runs) { run_ptr_.push_back(r.data); run_n_.push_back(r.n); }
    return esvo_ts_push_event_array(cs_->ctx(), cam_, run_ptr_.data(), run_n_.data(), (int)runs.size()) == ESVO_OK;
  }
  // events in this camera's log since construction / clearEventQueue (those a hot-pixel mask kept): the `total` of the
  // event windows read from the log (esvo_events_window_dev, esvo_events_lower_bound_dev)
  size_t eventsPushed() const {
    int64_t total = 0;
    esvo_ts_events_pushed(cs_->ctx(), cam_, &total);
    return (size_t)total;
  }
  // syncCallback -> createTimeSurfaceAtTime (TimeSurface.cpp:52-152,293-311); time_surface_out: H*W mono8 or nullptr
  bool createTimeSurfaceAtTime(int64_t external_sync_time_ns, uint8_t* time_surface_out) {
    return esvo_ts_build(cs_->ctx(), cam_, external_sync_time_ns, nullptr, time_surface_out) == ESVO_OK;
  }
  void clearEventQueue() { esvo_ts_reset(cs_->ctx(), cam_); }
  // The reference tolerates stamps that arrive out of order (its insertion sort then re-queues events_.back(),
  // TimeSurface.cpp:410-422).  Off by default here (drivers deliver ordered packets; saves two kernels per push);
  // switch it on for sources that do not guarantee ordering -- results are then identical to the reference's.
  bool setUnorderedInput(bool enable) { return esvo_ts_set_unordered_input(cs_->ctx(), cam_, enable ? 1 : 0) == ESVO_OK; }
 private:
  esvo::CameraSystem::Ptr cs_;
  int cam_;
  std::vector<uint16_t> x_, y_;
  std::vector<int64_t> t_;
  std::vector<uint8_t> p_;
  std::vector<const uint8_t*> run_ptr_;
  std::vector<size_t> run_n_;
};
}  // namespace esvo_time_surface

namespace esvo_core {
namespace core {
using esvo::CameraSystem;
using esvo::DepthPoint;
using esvo::EventMatchPair;

// core::EventBM (EventBM.h:27-60).  Patch size / disparity range / step / threshold come from the params the
// CameraSystem was created with (the reference passes them to resetParameters from the same yaml).
class EventBM {
 public:
  explicit EventBM(CameraSystem::Ptr camSysPtr) : camSysPtr_(std::move(camSysPtr)) {}
  void createMatchProblem(esvo::StampedTimeSurfaceObs* pStampedTsObs, esvo::StampTransformationMap* pSt_map,
                          std::vector<esvo::Event*>* pvEventsPtr) {
    pStampedTsObs_ = pStampedTsObs; pSt_map_ = pSt_map;
    ex_.clear(); ey_.clear(); et_.clear();
    for (auto* e : *pvEventsPtr) { ex_.push_back(e->x); ey_.push_back(e->y); et_.push_back(e->ts); }
  }
  void match_all_HyperThread(std::vector<EventMatchPair>& vEMP) {
    vEMP.clear();
    if (!pStampedTsObs_ || !pSt_map_) return;
    const auto& obs = pStampedTsObs_->second;
    if (esvo_set_ts_pair(camSysPtr_->ctx(), obs.left, obs.right, obs.tr_.data()) != ESVO_OK) return;
    const auto [pt, poses] = esvo::detail::stampsAndPoses(*pSt_map_);
    vEMP.resize(ex_.size());
    size_t n = vEMP.size();
    if (esvo_bm_match(camSysPtr_->ctx(), ex_.data(), ey_.data(), et_.data(), ex_.size(), pt.data(), poses.data(), pt.size(),
                      vEMP.data(), &n, &n_evals_) != ESVO_OK) n = 0;
    vEMP.resize(n);
  }
  void match_all_SingleThread(std::vector<EventMatchPair>& vEMP) { match_all_HyperThread(vEMP); }
  uint64_t n_evals_ = 0;
 private:
  CameraSystem::Ptr camSysPtr_;
  esvo::StampedTimeSurfaceObs* pStampedTsObs_ = nullptr;
  esvo::StampTransformationMap* pSt_map_ = nullptr;
  std::vector<uint16_t> ex_, ey_;
  std::vector<int64_t> et_;
};

enum DepthProblemType { ANALYTICAL, NUMERICAL };
// core::DepthProblemSolver (DepthProblemSolver.h:35-60)
class DepthProblemSolver {
 public:
  DepthProblemSolver(CameraSystem::Ptr& camSysPtr, DepthProblemType dpType = NUMERICAL) : camSysPtr_(camSysPtr), dpType_(dpType) {}
  void solve(std::vector<EventMatchPair>* pvEMP, esvo::StampedTimeSurfaceObs* pStampedTsObs, std::vector<DepthPoint>& vdp) {
    vdp.clear();
    if (dpType_ != NUMERICAL || !pvEMP || pvEMP->empty()) return;   // the reference exit(-1)s on ANALYTICAL
    const auto& obs = pStampedTsObs->second;
    if (esvo_set_ts_pair(camSysPtr_->ctx(), obs.left, obs.right, obs.tr_.data()) != ESVO_OK) return;
    vdp.resize(pvEMP->size());
    size_t n = vdp.size();
    if (esvo_depth_solve(camSysPtr_->ctx(), pvEMP->data(), pvEMP->size(), vdp.data(), &n, &n_evals_) != ESVO_OK) n = 0;
    vdp.resize(n);
  }
  void pointCulling(std::vector<DepthPoint>& vdp, double std_variance_threshold, double cost_threshold,
                    double invDepth_min_range, double invDepth_max_range) {
    size_t n = vdp.size();
    if (esvo_depth_cull(camSysPtr_->ctx(), vdp.data(), &n, std_variance_threshold, cost_threshold, invDepth_min_range,
                        invDepth_max_range) == ESVO_OK)
      vdp.resize(n);
  }
  DepthProblemType getProblemType() { return dpType_; }
  uint64_t n_evals_ = 0;
 private:
  CameraSystem::Ptr camSysPtr_;
  DepthProblemType dpType_;
};

// container::DepthFrame: the fused map lives on the device inside the ctx; this handle carries its pose.
struct DepthFrame {
  using Ptr = std::shared_ptr<DepthFrame>;
  esvo::Pose T_world_frame_{};
  size_t id_ = 0;
  bool fresh_ = true;   // a newly constructed DepthFrame starts from an empty map (esvo_Mapping.cpp:268-272)
  void setTransformation(const esvo::Pose& T) { T_world_frame_ = T; }
  void setId(size_t id) { id_ = id; }
};

// core::DepthFusion (DepthFusion.h:21-59)
class DepthFusion {
 public:
  explicit DepthFusion(CameraSystem::Ptr& camSysPtr) : camSysPtr_(camSysPtr) {}
  int update(std::vector<DepthPoint>& dp_obs, DepthFrame::Ptr& df, int fusion_radius) {
    int nf = 0;
    if (esvo_fuse(camSysPtr_->ctx(), dp_obs.data(), dp_obs.size(), df->T_world_frame_.data(), fusion_radius, df->fresh_ ? 1 : 0,
                  &nf) != ESVO_OK)
      return 0;
    df->fresh_ = false;
    return nf;
  }
  // naive_propagation (DepthFusion.cpp:232-288): nearest wins, no fusion -- the accumulation of the MVStereo comparison modes
  void naive_propagation(std::vector<DepthPoint>& dp_obs, DepthFrame::Ptr& df) {
    if (esvo_naive_propagate(camSysPtr_->ctx(), dp_obs.data(), dp_obs.size(), df->T_world_frame_.data(), df->fresh_ ? 1 : 0) == ESVO_OK)
      df->fresh_ = false;
  }
  // DepthMap::clean (SmartGrid.h:222-243) and the element list, exposed here because the map is ctx-resident
  void clean(double var_threshold, double age_threshold, double range_max, double range_min) {
    esvo_map_clean(camSysPtr_->ctx(), var_threshold, age_threshold, range_max, range_min);
  }
  void getElements(std::vector<DepthPoint>& out) {
    out.resize((size_t)camSysPtr_->width_ * camSysPtr_->height_);
    size_t n = out.size();
    if (esvo_map_download(camSysPtr_->ctx(), out.data(), &n) != ESVO_OK) n = 0;
    out.resize(n);
  }
 private:
  CameraSystem::Ptr camSysPtr_;
};

// core::DepthRegularization (DepthRegularization.h:20)
class DepthRegularization {
 public:
  explicit DepthRegularization(CameraSystem::Ptr& camSysPtr) : camSysPtr_(camSysPtr) {}
  void apply() { esvo_map_regularize(camSysPtr_->ctx()); }
 private:
  CameraSystem::Ptr camSysPtr_;
};

// core::EventSlice (EventMatcher.h:17-28): a run of left events that shares one virtual-view pose
struct EventSlice {
  explicit EventSlice(double SLICE_THICKNESS = 2 * 1e-3) : SLICE_THICKNESS_(SLICE_THICKNESS) {}
  size_t numEvents_ = 0;
  double SLICE_THICKNESS_;
  int64_t t_median_ = 0;
  esvo::Pose transf_{};
  std::vector<esvo::Event*>::iterator it_begin_, it_end_;
};

// core::EventMatcher (EventMatcher.h:30-100): the event-to-event matcher of [26] the reference keeps for comparison.
class EventMatcher {
 public:
  EventMatcher(CameraSystem::Ptr camSysPtr, size_t numThread = 1, double Time_THRESHOLD = 10e-5, double EPIPOLAR_THRESHOLD = 0.5,
               double TS_NCC_THRESHOLD = 0.1, size_t patch_size_X = 25, size_t patch_size_Y = 5, size_t patch_intensity_threshold = 125,
               double patch_valid_ratio = 0.1)
      : camSysPtr_(std::move(camSysPtr)), NUM_THREAD_(numThread) {
    resetParameters(Time_THRESHOLD, EPIPOLAR_THRESHOLD, TS_NCC_THRESHOLD, patch_size_X, patch_size_Y, patch_intensity_threshold, patch_valid_ratio);
  }
  void resetParameters(double Time_THRESHOLD, double EPIPOLAR_THRESHOLD, double TS_NCC_THRESHOLD, size_t patch_size_X, size_t patch_size_Y,
                       size_t patch_intensity_threshold, double patch_valid_ratio) {
    prm_.time_threshold_s = Time_THRESHOLD; prm_.epipolar_threshold = EPIPOLAR_THRESHOLD; prm_.ts_ncc_threshold = TS_NCC_THRESHOLD;
    prm_.patch_size_x = (int32_t)patch_size_X; prm_.patch_size_y = (int32_t)patch_size_Y; prm_.num_thread = (int32_t)NUM_THREAD_; prm_._pad = 0;
    patch_intensity_threshold_ = patch_intensity_threshold; patch_valid_ratio_ = patch_valid_ratio;   // unused by the reference as well
  }
  void createMatchProblem(esvo::StampedTimeSurfaceObs* pTS_obs, std::vector<EventSlice>* vEventSlice_ptr, std::vector<esvo::Event*>* vEventPtr_cand) {
    pTS_obs_ = pTS_obs; pvEventSlice_ = vEventSlice_ptr; pvCandEventPtr_ = vEventPtr_cand;
  }
  void match_all_HyperThread(std::vector<EventMatchPair>& vEMP) {
    vEMP.clear();
    if (!pTS_obs_ || !pvEventSlice_ || !pvCandEventPtr_ || pvEventSlice_->empty()) return;
    const auto& obs = pTS_obs_->second;
    if (esvo_set_ts_pair(camSysPtr_->ctx(), obs.left, obs.right, obs.tr_.data()) != ESVO_OK) return;
    // the events of all slices are contiguous from the first slice's begin (match(), EventMatcher.cpp:233-251)
    std::vector<int32_t> counts; std::vector<double> poses; size_t total = 0;
    for (auto& es : *pvEventSlice_) { counts.push_back((int32_t)es.numEvents_); poses.insert(poses.end(), es.transf_.begin(), es.transf_.end()); total += es.numEvents_; }
    std::vector<uint16_t> lx, ly, rx, ry; std::vector<int64_t> lt, rt; std::vector<uint8_t> lp, rp;
    auto it = (*pvEventSlice_)[0].it_begin_;
    for (size_t i = 0; i < total; ++i, ++it) { lx.push_back((*it)->x); ly.push_back((*it)->y); lt.push_back((*it)->ts); lp.push_back((*it)->polarity); }
    for (auto* e : *pvCandEventPtr_) { rx.push_back(e->x); ry.push_back(e->y); rt.push_back(e->ts); rp.push_back(e->polarity); }
    vEMP.resize(total);
    size_t n = total;
    if (esvo_em_match(camSysPtr_->ctx(), &prm_, lx.data(), ly.data(), lt.data(), lp.data(), total, counts.data(), poses.data(), counts.size(),
                      rx.data(), ry.data(), rt.data(), rp.data(), rx.size(), vEMP.data(), &n, &n_evals_) != ESVO_OK)
      n = 0;
    vEMP.resize(n);
  }
  // plain event order.  (The reference's single-thread walk additionally stops one event short of every slice's end,
  // EventMatcher.cpp:165-183; esvo_MVStereo only calls the HyperThread form, so that quirk is not reproduced.)
  void match_all_SingleThread(std::vector<EventMatchPair>& vEMP) {
    const int32_t nt = prm_.num_thread; prm_.num_thread = 1; match_all_HyperThread(vEMP); prm_.num_thread = nt;
  }
  uint64_t n_evals_ = 0;
 private:
  CameraSystem::Ptr camSysPtr_;
  size_t NUM_THREAD_;
  esvo_em_params prm_{};
  size_t patch_intensity_threshold_ = 125; double patch_valid_ratio_ = 0.1;
  esvo::StampedTimeSurfaceObs* pTS_obs_ = nullptr;
  std::vector<EventSlice>* pvEventSlice_ = nullptr;
  std::vector<esvo::Event*>* pvCandEventPtr_ = nullptr;
};

// core::RefFrame / CurFrame (RegProblemLM.h:58-74).  on_device_: the cloud is the one adopted on the device
// (esvo_track_adopt_map_dev) instead of vPointXYZ_.
struct RefFrame { int64_t t_ = 0; std::vector<float> vPointXYZ_; /* n*3, world frame; permuted in place */ esvo::Pose tr_{}; bool on_device_ = false; };
struct CurFrame { int64_t t_ = 0; const uint8_t* ts_left = nullptr; esvo::Pose tr_{}; size_t numEventsSinceLastObs_ = 0; };
struct LM_statics { size_t nPoints_ = 0, nfev_ = 0, nIter_ = 0; };
enum RegProblemType { REG_NUMERICAL, REG_ANALYTICAL };

// core::RegProblemSolverLM (RegProblemSolverLM.h:37-50)
class RegProblemSolverLM {
 public:
  RegProblemSolverLM(CameraSystem::Ptr& camSysPtr, RegProblemType rpType = REG_ANALYTICAL) : camSysPtr_(camSysPtr), rpType_(rpType) {}
  bool resetRegProblem(RefFrame* ref, CurFrame* cur) {
    cur_ = cur;
    int rc = ref->on_device_ ? esvo_track_reset_dev(camSysPtr_->ctx(), ref->tr_.data(), cur->tr_.data(), cur->ts_left)
                             : esvo_track_reset(camSysPtr_->ctx(), ref->vPointXYZ_.data(), ref->vPointXYZ_.size() / 3, ref->tr_.data(),
                                                cur->tr_.data(), cur->ts_left);
    lmStatics_ = LM_statics();
    return rc == ESVO_OK;   // 1 = not enough points in the local map -> the system re-initialises
  }
  bool solve_numerical() { return solve(0); }
  bool solve_analytical() { return solve(1); }
  LM_statics lmStatics_;
 private:
  bool solve(int analytical) {
    esvo_lm_stats st{};
    if (!cur_ || esvo_track_solve(camSysPtr_->ctx(), analytical, cur_->tr_.data(), &st) != ESVO_OK) return false;
    lmStatics_.nPoints_ = (size_t)st.n_points; lmStatics_.nfev_ = (size_t)st.nfev; lmStatics_.nIter_ = (size_t)st.n_iter;
    return true;
  }
  CameraSystem::Ptr camSysPtr_;
  RegProblemType rpType_;
  CurFrame* cur_ = nullptr;
};

}  // namespace core

// The event front-end of esvo_Mapping::dataTransferring (esvo_Mapping.cpp:536-603), host logic feeding the hot path:
//  * selectCloseEvents: the newest-first, at most PROCESS_EVENT_NUM left events with stamps in
//    [t_end - 10*BM_half_slice_thickness, t_end)  (:562-575; events_left_ is time-ordered);
//  * samplePoseStamps: the virtual-view stamps t_begin, t_begin + 0.05*BM_half_slice_thickness, ... <= t_end at
//    which the node looks up tf poses to fill st_map_ (:585-599).
// Both use the reference's ros::Time <-> double conversions (toSec() compares, Time(double) construction).
namespace frontend {
inline double toSec(int64_t ns) { int64_t s = ns / 1000000000LL, n = ns % 1000000000LL; if (n < 0) { n += 1000000000LL; --s; } return (double)s + 1e-9 * (double)n; }
inline int64_t fromSec(double t) {   // ros::Time(double): sec = floor(t), nsec = round((t - sec) * 1e9), carry on overflow
  int64_t sec = (int64_t)std::floor(t);
  int64_t nsec = (int64_t)std::llround((t - (double)sec) * 1e9);
  sec += nsec / 1000000000LL; nsec %= 1000000000LL;
  return sec * 1000000000LL + nsec;
}
// tools::EventBuffer_lower_bound (utils.h:50-55) over a time-ordered, random-access buffer of esvo::Event: the first event
// whose stamp is not before t_ns.  It compares toSec() DOUBLES, so stamps that share a double are equal.
template <class Buffer>
inline size_t lowerBound(const Buffer& events, int64_t t_ns) {
  const double ts = toSec(t_ns);
  size_t lo = 0, hi = events.size();
  while (lo < hi) { size_t mid = (lo + hi) / 2; if (toSec(events[mid].ts) < ts) lo = mid + 1; else hi = mid; }
  return lo;
}
// The start of a window of window_s seconds that ends at t_end (:542,563): ros::Time(max(0, t_end.toSec() - window_s))
inline int64_t windowBegin(int64_t t_end_ns, double window_s) { return fromSec(std::max(0.0, toSec(t_end_ns) - window_s)); }
namespace detail {
// The walk of dataTransferring's windows: from lower_bound(t_end) back to, not including, lower_bound(windowBegin(t_end,
// window_s)), at most `budget` events, newest first (:547-551,570-574).  When no event is at/after t_end (the observation
// stamp is newer than the whole buffer -- the common case online) the reference's first push is deque::end()._M_cur, one
// slot past the newest event (UB: an unconstructed event); it then still walks back over the newest valid events.  We skip
// only that slot but keep its place in the budget.
template <class Buffer>
inline void walkWindow(Buffer& events, int64_t t_end_ns, double window_s, size_t budget, std::vector<esvo::Event*>& out) {
  out.clear();
  if (events.empty()) return;
  size_t ev_end = lowerBound(events, t_end_ns);
  const size_t ev_begin = lowerBound(events, windowBegin(t_end_ns, window_s));
  if (ev_end == events.size() && ev_end != ev_begin && budget > 0) { --ev_end; --budget; }
  while (ev_end != ev_begin && out.size() < budget) { out.push_back(&events[ev_end]); --ev_end; }
}
}  // namespace detail
// events_left: a time-ordered std::vector or std::deque (the node's EventQueue) of esvo::Event
template <class EventBuffer>
inline void selectCloseEvents(EventBuffer& events_left, int64_t t_end_ns, double BM_half_slice_thickness, size_t PROCESS_EVENT_NUM,
                              std::vector<esvo::Event*>& vCloseEventsPtr_left) {
  detail::walkWindow(events_left, t_end_ns, 10 * BM_half_slice_thickness, PROCESS_EVENT_NUM, vCloseEventsPtr_left);
}
//  * selectSGMEvents: the INITIALIZATION branch of dataTransferring (:538-552) -- window 2*BM_half_slice_thickness and
//    `<=` instead of `<` on the count (one event more than PROCESS_EVENT_NUM).
template <class EventBuffer>
inline void selectSGMEvents(EventBuffer& events_left, int64_t t_end_ns, double BM_half_slice_thickness, size_t PROCESS_EVENT_NUM,
                            std::vector<esvo::Event*>& vEventsPtr_left_SGM) {
  detail::walkWindow(events_left, t_end_ns, 2 * BM_half_slice_thickness, PROCESS_EVENT_NUM + 1, vEventsPtr_left_SGM);
}
inline std::vector<int64_t> samplePoseStamps(int64_t t_end_ns, double BM_half_slice_thickness) {
  std::vector<int64_t> out;
  const double t_end = toSec(t_end_ns);
  int64_t t_tmp = windowBegin(t_end_ns, 10 * BM_half_slice_thickness);
  while (toSec(t_tmp) <= t_end) { out.push_back(t_tmp); t_tmp = fromSec(toSec(t_tmp) + 0.05 * BM_half_slice_thickness); }
  return out;
}
//  * queueEvents: eventsCallback's EventQueue (esvo_Mapping.cpp:669-703, esvo_Tracking.cpp:294-321, esvo_MVStereo.cpp:
//    746-790): each event is insertion-sorted in behind the queued ones with a stamp not above its own, then the oldest
//    events above max_length are dropped.
inline void queueEvents(std::deque<esvo::Event>& EQ, const std::vector<esvo::Event>& events, size_t max_length) {
  for (const esvo::Event& e : events) {
    EQ.push_back(e);
    long i = (long)EQ.size() - 2;
    while (i >= 0 && EQ[(size_t)i].ts > e.ts) { EQ[(size_t)i + 1] = EQ[(size_t)i]; --i; }
    EQ[(size_t)(i + 1)] = e;
  }
  if (EQ.size() > max_length) EQ.erase(EQ.begin(), EQ.begin() + (long)(EQ.size() - max_length));
}
//  * createDenoisingMask / extractDenoisedEvents (esvo_Mapping.cpp:1046-1072, bDenoising_): binary event map of ALL
//    window events -> cv::medianBlur 3x3 (on a 0/255 image: a pixel survives iff at least 5 of its 3x3 neighbours,
//    borders replicated, carry an event) -> keep the close events that sit on surviving pixels, at most maxNum.
inline void createDenoisingMask(const std::vector<esvo::Event*>& vAllEventsPtr, std::vector<uint8_t>& mask, size_t row, size_t col) {
  std::vector<uint8_t> eventMap(row * col, 0);                       // Visualization::plot_eventMap (Visualization.cpp:96-104)
  for (const esvo::Event* e : vAllEventsPtr) if (e->x < col && e->y < row) eventMap[(size_t)e->y * col + e->x] = 255;
  mask.assign(row * col, 0);
  for (size_t y = 0; y < row; ++y)
    for (size_t x = 0; x < col; ++x) {
      int on = 0;
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const size_t yy = (size_t)std::min<long>(std::max<long>((long)y + dy, 0), (long)row - 1);
          const size_t xx = (size_t)std::min<long>(std::max<long>((long)x + dx, 0), (long)col - 1);
          on += eventMap[yy * col + xx] != 0;
        }
      mask[y * col + x] = on >= 5 ? 255 : 0;
    }
}
inline void extractDenoisedEvents(const std::vector<esvo::Event*>& vCloseEventsPtr, std::vector<esvo::Event*>& vEdgeEventsPtr,
                                  const std::vector<uint8_t>& mask, size_t col, size_t maxNum) {
  vEdgeEventsPtr.reserve(vCloseEventsPtr.size());
  for (esvo::Event* e : vCloseEventsPtr) {
    if (vEdgeEventsPtr.size() >= maxNum) break;
    if (mask[(size_t)e->y * col + e->x] == 255) vEdgeEventsPtr.push_back(e);
  }
}
//  * denoise: the denoising step of MappingAtTime (esvo_Mapping.cpp:282-304, esvo_MVStereo.cpp:385-405): with bDenoising the
//    mask of all window events keeps at most maxNum of the close events, without it the first maxNum of them are kept.
inline void denoise(const std::vector<esvo::Event*>& vAllEventsPtr, const std::vector<esvo::Event*>& vCloseEventsPtr, bool bDenoising,
                    size_t row, size_t col, size_t maxNum, std::vector<esvo::Event*>& vDenoisedEventsPtr) {
  vDenoisedEventsPtr.clear();
  if (bDenoising) {
    std::vector<uint8_t> mask;
    createDenoisingMask(vAllEventsPtr, mask, row, col);
    extractDenoisedEvents(vCloseEventsPtr, vDenoisedEventsPtr, mask, col, maxNum);
  } else {
    vDenoisedEventsPtr.assign(vCloseEventsPtr.begin(), vCloseEventsPtr.begin() + (long)std::min(vCloseEventsPtr.size(), maxNum));
  }
}
//  * the local-map hand-off of publishPointCloud (esvo_Mapping.cpp:909-953): p_world = R p_cam + t as pcl::PointXYZ
//    (f32 x,y,z) in DepthMap iteration order; `near` additionally keeps ||p_cam|| < visualize_range (:930-931).
//    The result is what RefFrame::vPointXYZ_ / esvo_track_reset consume on the tracking side (esvo_Tracking.cpp:202-234).
inline void packPointCloud(const std::vector<esvo::DepthPoint>& elems, const esvo::Pose& T_world_result, std::vector<float>& xyz,
                           std::vector<float>* xyz_near = nullptr, double visualize_range = 0.0) {
  xyz.clear(); xyz.reserve(3 * elems.size());
  if (xyz_near) xyz_near->clear();
  const double* T = T_world_result.data();
  for (const esvo::DepthPoint& d : elems) {
    const double* p = d.p_cam;
    const double w[3] = {T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3], T[4] * p[0] + T[5] * p[1] + T[6] * p[2] + T[7],
                         T[8] * p[0] + T[9] * p[1] + T[10] * p[2] + T[11]};
    for (int k = 0; k < 3; ++k) xyz.push_back((float)w[k]);
    if (xyz_near && std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]) < visualize_range)
      for (int k = 0; k < 3; ++k) xyz_near->push_back((float)w[k]);
  }
}
//  * eventSlicingForEM (esvo_MVStereo.cpp:1008-1040): cuts the time-ordered left events of [t_lowBound, t_upBound) into
//    floor((t_up - t_low) / EM_Slice_Thickness) slices; a slice runs from its first event to lower_bound(first stamp +
//    thickness) INCLUSIVE, the next one starts behind it; its pose is the trajectory at the median event's stamp.
template <class PoseAt>
inline void eventSlicingForEM(std::vector<esvo::Event*>& vEventsPtr_left, int64_t t_lowBound_ns, int64_t t_upBound_ns, double EM_Slice_Thickness,
                              PoseAt&& getPoseAt, std::vector<core::EventSlice>& eventSlices) {
  eventSlices.clear();
  if (vEventsPtr_left.empty()) return;
  const size_t numSlice = (size_t)std::floor((toSec(t_upBound_ns) - toSec(t_lowBound_ns)) / EM_Slice_Thickness);
  auto it_tmp = vEventsPtr_left.begin();
  for (size_t i = 0; i < numSlice; ++i) {
    core::EventSlice es(EM_Slice_Thickness);
    es.it_begin_ = it_tmp;
    const double t_end = toSec(fromSec(toSec((*it_tmp)->ts) + es.SLICE_THICKNESS_));
    es.it_end_ = std::lower_bound(vEventsPtr_left.begin(), vEventsPtr_left.end(), t_end,
                                  [](const esvo::Event* e, double t) { return toSec(e->ts) < t; });   // tools::EventVecPtr_lower_bound (utils.h:43-48)
    if (es.it_end_ == vEventsPtr_left.end()) --es.it_end_;
    es.numEvents_ = (size_t)std::distance(es.it_begin_, es.it_end_) + 1;
    auto it_median = es.it_begin_;
    std::advance(it_median, es.numEvents_ / 2);
    es.t_median_ = (*it_median)->ts;
    getPoseAt(es.t_median_, es.transf_);
    eventSlices.push_back(es);
    it_tmp = es.it_end_;
    ++it_tmp;
    if (it_tmp == vEventsPtr_left.end()) break;
  }
}
//  * selectEMEvents: the event-matching branch of esvo_MVStereo::dataTransferring (esvo_MVStereo.cpp:579-609), one event
//    queue at a time.  The window is [lower_bound(t_low), lower_bound(t_up) - 1): the walk stops one event short of
//    lower_bound(t_up), and `<=` on the count lets EM_numEventMatching + 1 events through.  Returns false where the
//    reference returns "no events": lower_bound(t_low) == lower_bound(t_up) - 1.  With no event at all in [t_low, t_up)
//    the reference decrements past lower_bound(t_low) (or past begin()) and walks out of the window (undefined); that case
//    is answered the same way, false and nothing selected.
template <class EventBuffer>
inline bool selectEMEvents(EventBuffer& events, int64_t t_low_ns, int64_t t_up_ns, size_t EM_numEventMatching,
                           std::vector<esvo::Event*>& vEventsPtr) {
  vEventsPtr.clear();
  size_t lo = lowerBound(events, t_low_ns);
  const size_t up = lowerBound(events, t_up_ns);
  if (up <= lo + 1) return false;
  while (lo != up - 1 && vEventsPtr.size() <= EM_numEventMatching) vEventsPtr.push_back(&events[lo++]);
  return true;
}
//  * findObservation: the observation of dataTransferring (esvo_Mapping.cpp:501-534, esvo_MVStereo.cpp:560-576) -- the
//    newest history entry but one, walking back to the oldest, the first one poseAt gives a pose for (then in tr).  Returns
//    history.end() when there is none.  The history holds at least two entries.
template <class Entry, class PoseAt>
inline typename std::map<int64_t, Entry>::const_iterator findObservation(const std::map<int64_t, Entry>& history, PoseAt&& poseAt,
                                                                         esvo::Pose& tr) {
  auto it = std::next(history.rbegin());                 // in case the tf is behind the most current TS
  for (;; ++it) {
    tr = esvo::Pose{};
    if (poseAt(it->first, tr)) return std::prev(it.base());
    if (it->first == history.begin()->first) return history.end();
  }
}
}  // namespace frontend
}  // namespace esvo_core

namespace esvo {
// The tf::Transformer(true, ros::Duration(100.0)) the nodes keep (esvo_Mapping.cpp:140, esvo_Tracking.cpp:58,
// esvo_MVStereo.cpp:142), filled by stampedPoseCallback and read by getPoseAt.  Restates the tf2 TimeCache behaviour the
// nodes rely on (DESIGN.md section 2):
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
  // tf's getLatestCommonTime for the one world -> dvs link: the newest stamp; false (t untouched) when the buffer is empty
  bool latestCommonTime(int64_t& t_ns) const {
    if (s_.empty()) return false;
    t_ns = s_.back().t;
    return true;
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

// esvo_core::esvo_Mapping::MappingAtTime (esvo_Mapping.cpp:261-399) as one call with device-resident hand-off.
class esvo_Mapping {
 public:
  explicit esvo_Mapping(esvo::CameraSystem::Ptr cs) : cs_(std::move(cs)) {}
  struct Counters { uint64_t n_events, n_seeds, n_solved, n_culled, n_fusions, bm_evals, lm_evals, map_size; };
  bool MappingAtTime(const esvo::StampedTimeSurfaceObs& TS_obs, const std::vector<esvo::Event*>& vCloseEventsPtr_left,
                     const esvo::StampTransformationMap& st_map, Counters* out = nullptr) {
    return mapping(TS_obs, &vCloseEventsPtr_left, st_map, out);
  }
  // InitializationAtTime (esvo_Mapping.cpp:433-492).  The SGM stays where it is -- the node's
  //   sgbm_->compute(TS_left, TS_right, dispMap)       (cv::StereoSGBM(0,48,11,968,3872,-1,0,11), esvo_Mapping.cpp:101-108,444)
  // -- and its CV_16S result is passed in; everything downstream (edge mask AND disparity, DepthPoint creation,
  // naive_propagation into the new DepthFrame, first window vector) runs on the device.  Returns false like the
  // reference when fewer than INIT_SGM_DP_NUM_Threshold points survive.
  bool InitializationAtTime(const esvo::StampedTimeSurfaceObs& TS_obs, const int16_t* dispMap16,
                            const std::vector<esvo::Event*>& vEventsPtr_left_SGM, size_t INIT_SGM_DP_NUM_Threshold, size_t* n_points = nullptr) {
    std::vector<uint16_t> ex, ey;
    for (auto* e : vEventsPtr_left_SGM) { ex.push_back(e->x); ey.push_back(e->y); }
    size_t n = 0; int accepted = 0;
    if (esvo_init_from_disparity(cs_->ctx(), dispMap16, ex.data(), ey.data(), ex.size(), TS_obs.second.tr_.data(), INIT_SGM_DP_NUM_Threshold,
                                 &n, &accepted) != ESVO_OK)
      return false;
    if (n_points) *n_points = n;
    return accepted != 0;
  }
  // Same, with the SGM itself on the device as well (esvo_sgbm_compute: bit-exact restatement of cv::StereoSGBM MODE_SGBM with
  // the reference's parameters, esvo_Mapping.cpp:101-108) -- no OpenCV needed on the node side.
  bool InitializationAtTime(const esvo::StampedTimeSurfaceObs& TS_obs, const std::vector<esvo::Event*>& vEventsPtr_left_SGM,
                            size_t INIT_SGM_DP_NUM_Threshold, size_t* n_points = nullptr) {
    std::vector<int16_t> disp;
    if (!disparity(TS_obs, disp)) return false;
    return InitializationAtTime(TS_obs, disp.data(), vEventsPtr_left_SGM, INIT_SGM_DP_NUM_Threshold, n_points);
  }
  void reset() { esvo_mapping_reset(cs_->ctx()); }

  // ---- the node around MappingAtTime / InitializationAtTime: callbacks, dataTransferring and one pass of MappingLoop ----
  // (esvo_Mapping.cpp:179-259,494-605,669-762).  The ROS subscriptions become plain methods that fill the same buffers; the
  // tf look-up becomes a pose provider; ESVO_System_Status_ is the /ESVO_SYSTEM_STATUS value the owner keeps in sync.
  using PoseProvider = std::function<bool(int64_t /*stamp ns*/, esvo::Pose& /*T_world_dvs*/)>;   // getPoseAt (:646-667)
  void setPoseProvider(PoseProvider f) { getPoseAt_ = std::move(f); }
  // node parameters (constructor defaults of esvo_Mapping.cpp:77-92; cfg/mapping/*.yaml override them)
  size_t PROCESS_EVENT_NUM_ = 500, TS_HISTORY_LENGTH_ = 100, INIT_SGM_DP_NUM_Threshold_ = 500;
  double BM_half_slice_thickness_ = 0.001;
  bool bDenoising_ = false;
  std::string ESVO_System_Status_ = "INITIALIZATION";
  // eventsCallback (:669-703) for events_left_ / events_right_: insertion-sorted, capped at 3e6
  void eventsCallback(const std::vector<esvo::Event>& events, bool left) {
    frontend::queueEvents(left ? events_left_ : events_right_, events, MAX_EVENT_QUEUE_LENGTH);
  }
  static constexpr size_t MAX_EVENT_QUEUE_LENGTH = 3000000;
  // Device form: the left events are in camera 0's time-surface log on this context, total_left of them since it was reset
  // (esvo_time_surface::TimeSurface::eventsPushed).  events_left_ stays empty; dataTransferring then selects its window and the
  // denoised subset on the device (esvo_events_window_dev over the deque's place in the log, [max(0, total - 3e6), total)),
  // and InitializationAtTime / MappingAtTime run on that selection.  events_right_ is never read by the mapper.
  void eventsCallback(size_t total_left) { log_total_ = total_left; events_in_log_ = true; }
  // timeSurfaceCallback (:716-762): the stereo pair is copied into a history of TS_HISTORY_LENGTH_ entries
  void timeSurfaceCallback(int64_t stamp_ns, const uint8_t* time_surface_left, const uint8_t* time_surface_right) {
    const size_t n = (size_t)cs_->width_ * cs_->height_;
    TS_history_[stamp_ns] = TsPair{std::vector<uint8_t>(time_surface_left, time_surface_left + n),
                                   std::vector<uint8_t>(time_surface_right, time_surface_right + n), TS_id_++, false};
    while (TS_history_.size() > TS_HISTORY_LENGTH_) TS_history_.erase(TS_history_.begin());
  }
  // Device form: the pair just built on this context (both cameras at stamp_ns) goes into the device history
  // (esvo_ts_history_store_dev, reserved by the owner with TS_HISTORY_LENGTH_ pairs); the host history keeps the stamp only.
  bool timeSurfaceCallback(int64_t stamp_ns) {
    if (esvo_ts_history_store_dev(cs_->ctx(), stamp_ns) != ESVO_OK) return false;
    TS_history_[stamp_ns] = TsPair{{}, {}, TS_id_++, true};
    while (TS_history_.size() > TS_HISTORY_LENGTH_) TS_history_.erase(TS_history_.begin());
    return true;
  }
  // dataTransferring (:494-605).  Leaves TS_obs_ (second-newest entry with a pose; identity in INITIALIZATION), and
  // vEventsPtr_left_SGM_ (INITIALIZATION) or vALLEventsPtr_left_ / vCloseEventsPtr_left_ / st_map_ (WORKING).
  bool dataTransferring() {
    TS_obs_ = esvo::StampedTimeSurfaceObs(); has_obs_ = false;
    if (TS_history_.size() <= 10) return false;
    bool lost = false;   // a failed look-up took the status off WORKING: the walk stops there and dataTransferring fails (:521-527)
    esvo::Pose tr;
    const auto it = frontend::findObservation(TS_history_, [&](int64_t t, esvo::Pose& T) {
      if (ESVO_System_Status_ == "INITIALIZATION") { T = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; return true; }
      if (ESVO_System_Status_ != "WORKING") return false;
      if (getPoseAt_ && getPoseAt_(t, T)) return true;
      return lost = ESVO_System_Status_ != "WORKING";
    }, tr);
    if (lost || it == TS_history_.end()) return false;
    TS_obs_.first = it->first;
    TS_obs_.second.stored_ = it->second.stored;
    TS_obs_.second.left = it->second.stored ? nullptr : it->second.left.data();
    TS_obs_.second.right = it->second.stored ? nullptr : it->second.right.data();
    TS_obs_.second.id_ = it->second.id; TS_obs_.second.setTransformation(tr);
    has_obs_ = true;
    sel_on_device_ = false;
    if (ESVO_System_Status_ == "INITIALIZATION") {         // SGM (:537-552)
      if (events_in_log_) { if (!selectOnDevice(2 * BM_half_slice_thickness_, PROCESS_EVENT_NUM_ + 1, false, PROCESS_EVENT_NUM_ + 1)) return false; }
      else frontend::selectSGMEvents(events_left_, TS_obs_.first, BM_half_slice_thickness_, PROCESS_EVENT_NUM_, vEventsPtr_left_SGM_);
    }
    if (ESVO_System_Status_ == "WORKING") {                // BM (:554-603)
      if (events_in_log_) {                                // the walk and the denoising step (:282-304) in one device call
        if (!selectOnDevice(10 * BM_half_slice_thickness_, PROCESS_EVENT_NUM_, bDenoising_, PROCESS_EVENT_NUM_)) return false;
      } else {
        frontend::selectCloseEvents(events_left_, TS_obs_.first, BM_half_slice_thickness_, PROCESS_EVENT_NUM_, vCloseEventsPtr_left_);
        vALLEventsPtr_left_ = vCloseEventsPtr_left_;       // both are filled by the same walk (:569-574)
      }
      st_map_.clear();
      for (int64_t t : frontend::samplePoseStamps(TS_obs_.first, BM_half_slice_thickness_)) {
        esvo::Pose tr;
        if (getPoseAt_ && getPoseAt_(t, tr)) st_map_.push_back({t, tr});
        else if (ESVO_System_Status_ != "WORKING") return false;
      }
    }
    return true;
  }
  // What one pass of MappingLoop did.  ran: 0 nothing, 1 InitializationAtTime, 2 MappingAtTime; ok: the call's result;
  // cloud: the local map as publishPointCloud publishes it (world frame, at the observation's pose), if it did; with a stored
  // observation it is published on the device instead (esvo_map_publish_dev) and `cloud` stays empty.  cloud_points: its size.
  struct LoopResult {
    int ran = 0; bool ok = false; size_t n_sgm_points = 0; Counters ctr{};
    bool published = false; int64_t stamp = 0; esvo::Pose T_world_obs{}; std::vector<float> cloud; size_t cloud_points = 0;
  };
  // one pass of MappingLoop's body (:194-248) with publishMappingResults / publishPointCloud (:396-403,488-490,868-953) run in line
  bool MappingLoopOnce(LoopResult& res) {
    res = LoopResult();
    if (ESVO_System_Status_ == "TERMINATE" || TS_history_.size() < 10) return false;
    { auto _ = calls_.time("mapping.dataTransferring"); dataTransferring(); }
    if (!error_.empty() || !has_obs_) return false;
    if (ESVO_System_Status_ == "INITIALIZATION" || ESVO_System_Status_ == "RESET") {
      res.ran = 1;
      { auto _ = calls_.time("mapping.InitializationAtTime");
        res.ok = sel_on_device_ ? initializationOnSelection(&res.n_sgm_points)
                                : InitializationAtTime(TS_obs_, vEventsPtr_left_SGM_, INIT_SGM_DP_NUM_Threshold_, &res.n_sgm_points); }
      if (res.ok) { auto _ = calls_.time("mapping.publishMappingResults"); publishMappingResults(res); }
    }
    if (ESVO_System_Status_ == "WORKING") {
      res.ran = 2;
      if (!sel_on_device_) {                                 // the device form denoised in dataTransferring
        auto _ = calls_.time("mapping.denoising");
        frontend::denoise(vALLEventsPtr_left_, vCloseEventsPtr_left_, bDenoising_, (size_t)cs_->height_, (size_t)cs_->width_, PROCESS_EVENT_NUM_,
                          vDenoisedEventsPtr_left_);
      }
      { auto _ = calls_.time("mapping.MappingAtTime");
        res.ok = mapping(TS_obs_, sel_on_device_ ? nullptr : &vDenoisedEventsPtr_left_, st_map_, &res.ctr); }
      if (res.ok) { auto _ = calls_.time("mapping.publishMappingResults"); publishMappingResults(res); }
    }
    return res.ok;
  }
  // Number of vectors in the fusion window (dqvDepthPoints_.size()) and of points in them, read from the ctx.
  size_t fusionWindow(size_t* n_points = nullptr) {
    size_t k = 0, total = 0;
    for (;; ++k) {
      size_t n = 0;
      const int rc = esvo_window_download(cs_->ctx(), (int)k, nullptr, &n);
      if (rc != ESVO_OK && rc != ESVO_ERR_CAPACITY) break;
      total += n;
    }
    if (n_points) *n_points = total;
    return k;
  }
  esvo::StampedTimeSurfaceObs TS_obs_;
  std::vector<esvo::Event*> vEventsPtr_left_SGM_, vALLEventsPtr_left_, vCloseEventsPtr_left_, vDenoisedEventsPtr_left_;
  esvo::StampTransformationMap st_map_;
  esvo::CallTimes calls_;   // host time of each call MappingLoopOnce makes
  std::string error_;       // device form: why the log could not answer a window (MappingLoopOnce then returned false)
 private:
  // The device form of a dataTransferring window: the walk of selectCloseEvents / selectSGMEvents from lower_bound(t_obs) back
  // to lower_bound(frontend::windowBegin(t_obs, window)), at most `budget` events, then the denoising mask; at most max_keep
  // are kept.  The selection stays on the device.
  bool selectOnDevice(double window, size_t budget, bool denoise, size_t max_keep) {
    const int64_t t_begin = frontend::windowBegin(TS_obs_.first, window);
    const int64_t front = log_total_ > MAX_EVENT_QUEUE_LENGTH ? (int64_t)(log_total_ - MAX_EVENT_QUEUE_LENGTH) : 0;
    if (esvo_events_window_dev(cs_->ctx(), 0, front, t_begin, TS_obs_.first, budget, denoise ? 1 : 0, max_keep, &n_selected_) != ESVO_OK) {
      error_ = std::string("event window: ") + esvo_last_error(cs_->ctx());
      return false;
    }
    sel_on_device_ = true;
    return true;
  }
  // the SGM of InitializationAtTime (:444): cv::StereoSGBM(0, 48, 11, 968, 3872, -1, 0, 11) on the observation
  // (esvo_Mapping.cpp:101-108), on the device
  bool disparity(const esvo::StampedTimeSurfaceObs& TS_obs, std::vector<int16_t>& disp) {
    const int num_disparities = 16 * 3, block_size = 11;                       // esvo_Mapping.cpp:101-105
    disp.resize((size_t)cs_->width_ * cs_->height_);
    if (TS_obs.second.stored_ && !setObservation(TS_obs)) return false;      // a stored pair: the SGM reads the observation
    return esvo_sgbm_compute(cs_->ctx(), TS_obs.second.left, TS_obs.second.right, num_disparities, block_size, 8 * block_size * block_size,
                             32 * block_size * block_size, -1, 0, 11, disp.data()) == ESVO_OK;
  }
  bool initializationOnSelection(size_t* n_points) {
    std::vector<int16_t> disp;
    if (!disparity(TS_obs_, disp)) return false;
    size_t n = 0; int accepted = 0;
    if (esvo_init_from_disparity_selected_dev(cs_->ctx(), disp.data(), TS_obs_.second.tr_.data(), INIT_SGM_DP_NUM_Threshold_, &n, &accepted) != ESVO_OK)
      return false;
    if (n_points) *n_points = n;
    return accepted != 0;
  }
  // MappingAtTime on the host events, or with events == nullptr on the device selection of dataTransferring
  bool mapping(const esvo::StampedTimeSurfaceObs& TS_obs, const std::vector<esvo::Event*>* events, const esvo::StampTransformationMap& st_map,
               Counters* out) {
    if (!setObservation(TS_obs)) return false;
    std::vector<uint16_t> ex, ey; std::vector<int64_t> et;
    if (events) for (auto* e : *events) { ex.push_back(e->x); ey.push_back(e->y); et.push_back(e->ts); }
    const auto [pt, poses] = esvo::detail::stampsAndPoses(st_map);
    uint64_t c[8];
    const int rc = events ? esvo_mapping_at_time(cs_->ctx(), ex.data(), ey.data(), et.data(), ex.size(), pt.data(), poses.data(), pt.size(), c)
                          : esvo_mapping_at_time_selected_dev(cs_->ctx(), pt.data(), poses.data(), pt.size(), c);
    if (rc != ESVO_OK) return false;
    if (out) *out = Counters{c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7]};
    return true;
  }
  // the observation to the device: the stored pair by its stamp, or the host images (nullptr: the last builds)
  bool setObservation(const esvo::StampedTimeSurfaceObs& TS_obs) {
    const auto& obs = TS_obs.second;
    if (obs.stored_) return esvo_set_ts_pair_stored_dev(cs_->ctx(), TS_obs.first, obs.tr_.data()) == ESVO_OK;
    return esvo_set_ts_pair(cs_->ctx(), obs.left, obs.right, obs.tr_.data()) == ESVO_OK;
  }
  // publishMappingResults (:868-907): in INITIALIZATION always, in WORKING once the fusion window is full (CONST_FRAMES) or
  // holds more than half of maxNumFusionPoints (CONST_POINTS); publishPointCloud (:909-953) skips an empty cloud
  void publishMappingResults(LoopResult& res) {
    const esvo_params& p = cs_->params();
    bool publish = ESVO_System_Status_ == "INITIALIZATION";
    if (ESVO_System_Status_ == "WORKING") {
      size_t n_points = 0;
      const size_t n_frames = fusionWindow(&n_points);
      if (p.fusion_strategy == ESVO_FUSION_CONST_FRAMES) publish = n_frames == (size_t)p.max_num_fusion_frames;
      else publish = (double)n_points > 0.5 * (double)p.max_num_fusion_points;
    }
    if (!publish) return;
    if (TS_obs_.second.stored_) {                        // device form: the cloud stays on the device for the tracker
      if (esvo_map_publish_dev(cs_->ctx(), TS_obs_.second.tr_.data(), TS_obs_.first, &res.cloud_points) != ESVO_OK) res.cloud_points = 0;
    } else {
      std::vector<esvo::DepthPoint> elems((size_t)cs_->width_ * cs_->height_);
      size_t n = elems.size();
      if (esvo_map_download(cs_->ctx(), elems.data(), &n) != ESVO_OK) n = 0;
      elems.resize(n);
      frontend::packPointCloud(elems, TS_obs_.second.tr_, res.cloud);
      res.cloud_points = res.cloud.size() / 3;
    }
    if (res.cloud_points == 0) return;
    res.published = true; res.stamp = TS_obs_.first; res.T_world_obs = TS_obs_.second.tr_;
  }
  struct TsPair { std::vector<uint8_t> left, right; size_t id; bool stored; };   // stored: the images are in the device history
  esvo::CameraSystem::Ptr cs_;
  std::deque<esvo::Event> events_left_, events_right_;   // EventQueue (esvo_Mapping.h)
  size_t log_total_ = 0, n_selected_ = 0;                 // device form: left events in the log; size of the selection
  bool events_in_log_ = false, sel_on_device_ = false;
  std::map<int64_t, TsPair> TS_history_;
  size_t TS_id_ = 0;
  bool has_obs_ = false;
  PoseProvider getPoseAt_;
};

// The host half of the esvo_MVStereo node (esvo_MVStereo.cpp:179-237,552-880,1002-1039): the event queues, the
// time-surface history, the tf pose buffer fed by the stamped_pose topic, the three reset rules, getPoseAt, the per-mode
// dataTransferring windows and the BM denoising step of MappingAtTime.  Host logic only -- no device call, so it builds
// and is tested without the library; esvo_MVStereo below owns one and runs MappingAtTime on what it selects.
// Modes use esvo_MVStereo::eMVStereoMode numbering (0 EM, 1 BM, 2 EM + estimation, 3 BM + estimation, 4 SGM).
class MVStereoFrontEnd {
 public:
  MVStereoFrontEnd(int width, int height, int msm) : W_((size_t)width), H_((size_t)height), msm_(msm) {}
  // node parameters (constructor defaults of esvo_MVStereo.cpp:71-101; cfg/mvstereo/*.yaml override them)
  size_t PROCESS_EVENT_NUM_ = 500, TS_HISTORY_LENGTH_ = 100, EM_numEventMatching_ = 3000;
  double BM_half_slice_thickness_ = 0.001;
  bool bDenoising_ = false;
  bool marker_frame_ = false;   // dvs_frame_id "marker" (mvstereo_rpg.launch): getPoseAt appends T_marker_cam
  static constexpr size_t MAX_NUM_Event_INVOLVED = 10000;   // BM window cap (:639)

  // ---- callbacks.  Each returns true when its reset rule fired: reset() ran before the new data was added. ----
  // eventsCallback (:746-780): dt = first new stamp - newest queued stamp of the same queue; dt < 0 or >= 0.5 s resets.
  // Then insertion-sorted, capped at 3e6.  (The reference reads events[0] before its emptiness check; an empty packet
  // here changes nothing.)
  bool eventsCallback(const std::vector<esvo::Event>& events, bool left) {
    if (events.empty()) return false;
    bool was_reset = false;
    std::deque<esvo::Event>& EQ = left ? events_left_ : events_right_;
    if (!EQ.empty() && inconsistent(events[0].ts, EQ.back().ts)) { reset(); was_reset = true; }
    static constexpr size_t MAX_EVENT_QUEUE_LENGTH = 3000000;   // clearEventQueue (:782-790)
    frontend::queueEvents(EQ, events, MAX_EVENT_QUEUE_LENGTH);
    return was_reset;
  }
  // timeSurfaceCallback (:792-838): dt against the newest stamp in TS_history_; dt < 0 or >= 0.5 s resets.  The pair is
  // emplaced (a stamp already present keeps its old images), TS_id_ counts every call, the history keeps TS_HISTORY_LENGTH.
  bool timeSurfaceCallback(int64_t stamp_ns, const uint8_t* time_surface_left, const uint8_t* time_surface_right) {
    bool was_reset = false;
    if (!TS_history_.empty() && inconsistent(stamp_ns, TS_history_.rbegin()->first)) { reset(); was_reset = true; }
    const size_t n = W_ * H_;
    TS_history_.emplace(stamp_ns, TsPair{std::vector<uint8_t>(time_surface_left, time_surface_left + n),
                                         std::vector<uint8_t>(time_surface_right, time_surface_right + n), TS_id_});
    ++TS_id_;
    while (TS_history_.size() > TS_HISTORY_LENGTH_) TS_history_.erase(TS_history_.begin());
    return was_reset;
  }
  // stampedPoseCallback (:670-706): tf's latest common time is read first (tf2 writes it only on success, so after a
  // reset emptied the buffer the previous value stays); when it is not 0, dt = new stamp - it, and dt < 0 or >= 0.5 s
  // resets.  Then the pose goes into tf.
  bool stampedPoseCallback(int64_t stamp_ns, const esvo::Pose& T_world_dvs) {
    bool was_reset = false;
    tf_.latestCommonTime(tf_latest_common_time_);
    if (frontend::toSec(tf_latest_common_time_) != 0 && inconsistent(stamp_ns, tf_latest_common_time_)) { reset(); was_reset = true; }
    tf_.setTransform(stamp_ns, T_world_dvs);
    return was_reset;
  }
  // getPoseAt (:709-744): the tf pose; with dvs_frame_id "marker" the rpg rig's ground truth is the marker's pose and the
  // camera's is T_world_marker * T_marker_cam (the constant of :731-735).
  bool getPoseAt(int64_t t_ns, esvo::Pose& T) const {
    esvo::Pose Tm;
    if (!tf_.lookup(t_ns, Tm)) return false;
    if (!marker_frame_) { T = Tm; return true; }
    static constexpr double Mc[16] = {5.363262328777285e-01, -1.748374625145743e-02, -8.438296573030597e-01, -7.009849865398374e-02,
                                      8.433577587813513e-01, -2.821937531845164e-02, 5.366109927684415e-01, 1.881333563905305e-02,
                                      -3.319431623758162e-02, -9.994488408486204e-01, -3.897382049768972e-04, -6.966829200678797e-02,
                                      0, 0, 0, 1};
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) T[4 * r + c] = Tm[4 * r] * Mc[c] + Tm[4 * r + 1] * Mc[4 + c] + Tm[4 * r + 2] * Mc[8 + c] + Tm[4 * r + 3] * Mc[12 + c];
    return true;
  }
  // reset (:840-880): events, history, tf and TS_id_ here; the owner drops the map and the fusion window.  Not restated:
  // :862-864 re-arm the block matcher in modes 1 and 2 with the unclamped BM_min_disparity / BM_max_disparity, so after a
  // reset the reference's mode 1 searches [BM_min, BM_max] instead of the range the constructor clamps to the inverse-depth
  // limits (rpg: 1..40 instead of 4..40).  The disparity range is fixed when the context is made; here it stays clamped.
  void reset() {
    events_left_.clear(); events_right_.clear(); TS_history_.clear(); tf_.clear(); TS_id_ = 0;
    ++n_resets_;
  }

  // dataTransferring (:552-668).  TS_obs_: the newest entry but one, walking back to the oldest, that tf has a pose for.
  // Then the mode's window: EM frontend::selectEMEvents over [oldest TS, newest TS) on both queues (false: no events);
  // SGM frontend::selectSGMEvents (2 * BM_half_slice_thickness, `<=`); BM frontend::selectCloseEvents with the cap of
  // MAX_NUM_Event_INVOLVED (10 * BM_half_slice_thickness) into vALLEventsPtr_left_ and vCloseEventsPtr_left_, and the
  // virtual-view poses at frontend::samplePoseStamps, a stamp tf has no pose for being skipped.
  bool dataTransferring() {
    clearSelection();
    if (TS_history_.size() <= 10) return false;
    esvo::Pose tr;
    const auto it = frontend::findObservation(TS_history_, [&](int64_t t, esvo::Pose& T) { return getPoseAt(t, T); }, tr);
    if (it == TS_history_.end()) return false;
    TS_obs_.first = it->first;
    TS_obs_.second.left = it->second.left.data(); TS_obs_.second.right = it->second.right.data();
    TS_obs_.second.id_ = it->second.id; TS_obs_.second.setTransformation(tr);
    has_obs_ = true;
    if (msm_ == 0 || msm_ == 2) {
      t_lowBound_ = TS_history_.begin()->first; t_upBound_ = TS_history_.rbegin()->first;
      std::vector<esvo::Event*> l, r;
      if (!frontend::selectEMEvents(events_left_, t_lowBound_, t_upBound_, EM_numEventMatching_, l) ||
          !frontend::selectEMEvents(events_right_, t_lowBound_, t_upBound_, EM_numEventMatching_, r))
        return false;
      vEventsPtr_left_.swap(l); vEventsPtr_right_.swap(r);
    }
    if (msm_ == 4)
      frontend::selectSGMEvents(events_left_, TS_obs_.first, BM_half_slice_thickness_, PROCESS_EVENT_NUM_, vEventsPtr_left_SGM_);
    if (msm_ == 1 || msm_ == 3) {
      frontend::selectCloseEvents(events_left_, TS_obs_.first, BM_half_slice_thickness_, MAX_NUM_Event_INVOLVED, vCloseEventsPtr_left_);
      vALLEventsPtr_left_ = vCloseEventsPtr_left_;        // both are filled by the same walk (:642-647)
      for (int64_t t : frontend::samplePoseStamps(TS_obs_.first, BM_half_slice_thickness_)) {
        esvo::Pose tr;
        if (getPoseAt(t, tr)) st_map_.push_back({t, tr});
      }
    }
    return true;
  }
  // The BM branch of MappingAtTime before the matcher (:385-405): the denoising mask of all window events keeps at most
  // PROCESS_EVENT_NUM of the close events, or, without denoising, the first PROCESS_EVENT_NUM of them.
  void denoise() {
    frontend::denoise(vALLEventsPtr_left_, vCloseEventsPtr_left_, bDenoising_, H_, W_, PROCESS_EVENT_NUM_, vDenoisedEventsPtr_left_);
  }
  // The host part of one MappingLoop pass (:196-225): the TS_history_.size() >= 10 gate, dataTransferring, the skip when no
  // observation was loaded (TS_obs_ empty), and in BM modes the denoising.  true: MappingAtTime is due on TS_obs_ -- also
  // when dataTransferring returned false after loading the observation (the loop tests TS_obs_, not the return value).
  struct Pass { bool gated = false, transferred = false, has_obs = false; };
  bool prepare(Pass& p) {
    p = Pass();
    if (TS_history_.size() < 10) { clearSelection(); return false; }
    p.gated = true;
    p.transferred = dataTransferring();
    p.has_obs = has_obs_;
    if (!has_obs_) return false;
    if (msm_ == 1 || msm_ == 3) denoise();
    return true;
  }

  std::deque<esvo::Event> events_left_, events_right_;   // EventQueue
  struct TsPair { std::vector<uint8_t> left, right; size_t id; };
  std::map<int64_t, TsPair> TS_history_;
  size_t TS_id_ = 0, n_resets_ = 0;
  esvo::PoseBuffer tf_;
  int64_t tf_latest_common_time_ = 0;
  // what dataTransferring / denoise leave
  esvo::StampedTimeSurfaceObs TS_obs_;
  bool has_obs_ = false;
  std::vector<esvo::Event*> vEventsPtr_left_, vEventsPtr_right_, vEventsPtr_left_SGM_, vALLEventsPtr_left_, vCloseEventsPtr_left_,
      vDenoisedEventsPtr_left_;
  int64_t t_lowBound_ = 0, t_upBound_ = 0;
  esvo::StampTransformationMap st_map_;
  size_t W_, H_;
  int msm_;
 private:
  // The observation and every selection are cleared at the start of a pass: a pass without an observation leaves nothing
  // behind (the reference keeps the previous pass's pointers there, which nothing reads, and a reset leaves them dangling).
  void clearSelection() {
    TS_obs_ = esvo::StampedTimeSurfaceObs(); has_obs_ = false;
    for (auto* v : {&vEventsPtr_left_, &vEventsPtr_right_, &vEventsPtr_left_SGM_, &vALLEventsPtr_left_, &vCloseEventsPtr_left_,
                    &vDenoisedEventsPtr_left_})
      v->clear();
    st_map_.clear();
  }
  static bool inconsistent(int64_t t_new, int64_t t_old) {   // max_time_diff_before_reset_s = 0.5
    const double dt = frontend::toSec(t_new) - frontend::toSec(t_old);
    return dt < 0 || std::fabs(dt) >= 0.5;
  }
};

// esvo_core::esvo_MVStereo::MappingAtTime (esvo_MVStereo.cpp:239-520): the known-pose multi-view-stereo node the reference
// uses to compare five depth estimators on the same fusion back-end.  The node's dataTransferring (:544-668) fills the
// public input members below (front-end helpers: frontend::selectCloseEvents / samplePoseStamps / eventSlicingForEM);
// MappingAtTime then runs the selected mode on the device through the same ABI entry points the mapper uses.
class esvo_MVStereo {
 public:
  enum eMVStereoMode { PURE_EVENT_MATCHING, PURE_BLOCK_MATCHING, EM_PLUS_ESTIMATION, BM_PLUS_ESTIMATION, PURE_SEMI_GLOBAL_MATCHING };   // esvo_MVStereo.h:38-45
  using PoseProvider = std::function<bool(int64_t, esvo::Pose&)>;
  esvo_MVStereo(esvo::CameraSystem::Ptr cs, eMVStereoMode msm, size_t NUM_THREAD_MAPPING = 4)
      : node_(cs->width_, cs->height_, (int)msm), msm_(msm), em_(cs, NUM_THREAD_MAPPING), ebm_(cs), dpSolver_(cs), dFusor_(cs), dRegularizor_(cs), cs_(cs) {
    const esvo_params& p = cs_->params();
    em_.resetParameters(EM_Time_THRESHOLD_, EM_EPIPOLAR_THRESHOLD_, EM_TS_NCC_THRESHOLD_, (size_t)p.patch_size_x, (size_t)p.patch_size_y, 125, 0.1);   // :85-91
    maxNumFusionFrames_ = (size_t)p.max_num_fusion_frames; maxNumFusionPoints_ = (size_t)p.max_num_fusion_points;
  }
  void setPoseProvider(PoseProvider f) { getPoseAt_ = std::move(f); }
  void resetEMParameters(double thickness, double time_thr, double epi_thr, double ncc_thr) {
    EM_Slice_Thickness_ = thickness; EM_Time_THRESHOLD_ = time_thr; EM_EPIPOLAR_THRESHOLD_ = epi_thr; EM_TS_NCC_THRESHOLD_ = ncc_thr;
    const esvo_params& p = cs_->params();
    em_.resetParameters(time_thr, epi_thr, ncc_thr, (size_t)p.patch_size_x, (size_t)p.patch_size_y, 125, 0.1);
  }
  // ---- inputs, as dataTransferring leaves them (:544-668) ----
  esvo::StampedTimeSurfaceObs TS_obs_;
  std::vector<esvo::Event*> vEventsPtr_left_, vEventsPtr_right_;        // EM: all events of [t_lowBound_, t_upBound_)
  int64_t t_lowBound_ = 0, t_upBound_ = 0;
  std::vector<esvo::Event*> vCloseEventsPtr_left_;                       // BM: newest-first window events (already denoised / truncated)
  esvo::StampTransformationMap st_map_;
  std::vector<esvo::Event*> vEventsPtr_left_SGM_;                        // SGM: events that draw the edge mask
  // ---- results ----
  std::vector<esvo::EventMatchPair> vEMP_;
  std::deque<std::vector<esvo::DepthPoint>> dqvDepthPoints_;
  size_t numFusionCount_ = 0;

  bool MappingAtTime() {
    const esvo_params& p = cs_->params();
    core::DepthFrame::Ptr depthFramePtr_new = std::make_shared<core::DepthFrame>();             // :246-251
    depthFramePtr_new->setId(TS_obs_.second.id_);
    depthFramePtr_new->setTransformation(TS_obs_.second.tr_);
    depthFramePtr_ = depthFramePtr_new;
    vEMP_.clear();
    if (msm_ == PURE_EVENT_MATCHING || msm_ == EM_PLUS_ESTIMATION) {                            // :257-306
      std::vector<core::EventSlice> eventSlices;
      frontend::eventSlicingForEM(vEventsPtr_left_, t_lowBound_, t_upBound_, EM_Slice_Thickness_,
                                  [&](int64_t t, esvo::Pose& T) { return getPoseAt_ ? getPoseAt_(t, T) : false; }, eventSlices);
      em_.createMatchProblem(&TS_obs_, &eventSlices, &vEventsPtr_right_);
      em_.match_all_HyperThread(vEMP_);
      if (vEMP_.empty()) return false;
      if (msm_ == PURE_EVENT_MATCHING) { std::vector<esvo::DepthPoint> vdp; vEMP2vDP(vEMP_, vdp); return accumulateNaive(vdp); }
    }
    if (msm_ == PURE_SEMI_GLOBAL_MATCHING) {                                                    // :311-378
      std::vector<int16_t> dispMap((size_t)cs_->width_ * cs_->height_);
      if (esvo_set_ts_pair(cs_->ctx(), TS_obs_.second.left, TS_obs_.second.right, TS_obs_.second.tr_.data()) != ESVO_OK) return false;
      if (esvo_sgbm_compute(cs_->ctx(), nullptr, nullptr, (int)num_disparities_, (int)block_size_, (int)P1_, (int)P2_, -1, 0, 11, dispMap.data()) != ESVO_OK)
        return false;
      std::vector<esvo::DepthPoint> vdp_sgm;
      sgmPoints(dispMap, vdp_sgm);
      return accumulateNaive(vdp_sgm);
    }
    if (msm_ == PURE_BLOCK_MATCHING || msm_ == BM_PLUS_ESTIMATION) {                            // :383-431
      ebm_.createMatchProblem(&TS_obs_, &st_map_, &vCloseEventsPtr_left_);
      ebm_.match_all_HyperThread(vEMP_);
      if (msm_ == PURE_BLOCK_MATCHING) { std::vector<esvo::DepthPoint> vdp; vEMP2vDP(vEMP_, vdp); return accumulateNaive(vdp); }
    }
    // EM_PLUS_ESTIMATION / BM_PLUS_ESTIMATION: nonlinear optimisation, culling, fusion, clean, regularisation (:437-507)
    std::vector<esvo::DepthPoint> vdp;
    dpSolver_.solve(&vEMP_, &TS_obs_, vdp);
    dpSolver_.pointCulling(vdp, p.stdvar_vis_threshold, p.residual_vis_threshold * p.residual_vis_threshold * p.patch_size_x * p.patch_size_y,
                           p.invdepth_min_range, p.invdepth_max_range);
    dqvDepthPoints_.push_back(vdp);
    if (p.fusion_strategy == ESVO_FUSION_CONST_POINTS) {
      auto total = [&] { size_t n = 0; for (auto& v : dqvDepthPoints_) n += v.size(); return n; };
      while ((double)total() > 1.5 * (double)maxNumFusionPoints_) dqvDepthPoints_.pop_front();
    } else {
      while (dqvDepthPoints_.size() > maxNumFusionFrames_) dqvDepthPoints_.pop_front();
    }
    numFusionCount_ = 0;
    for (auto it = dqvDepthPoints_.rbegin(); it != dqvDepthPoints_.rend(); ++it) numFusionCount_ += (size_t)dFusor_.update(*it, depthFramePtr_, p.fusion_radius);
    dFusor_.clean(p.stdvar_vis_threshold * p.stdvar_vis_threshold, p.age_vis_threshold, p.invdepth_max_range, p.invdepth_min_range);
    if (p.regularization) dRegularizor_.apply();
    return true;
  }
  // vEMP2vDP (:1072-1097)
  void vEMP2vDP(std::vector<esvo::EventMatchPair>& vEMP, std::vector<esvo::DepthPoint>& vdp) {
    vdp.resize(vEMP.size());
    if (esvo_seeds_to_points(cs_->ctx(), vEMP.data(), vEMP.size(), vdp.data()) != ESVO_OK) vdp.clear();
  }
  void getElements(std::vector<esvo::DepthPoint>& out) { dFusor_.getElements(out); }
  void reset() { dqvDepthPoints_.clear(); }

  // ---- the node around MappingAtTime: callbacks, getPoseAt, dataTransferring, one pass of MappingLoop and the publishers
  // (esvo_MVStereo.cpp:179-237,552-880,960-1055).  The host logic is node_ (MVStereoFrontEnd); a reset it reports also
  // empties the map and drops the fusion window, as reset() (:840-880) does with depthFramePtr_ and dqvDepthPoints_.
  // The owner sets node_'s parameters and points the pose provider at getPoseAt (the EM slices look their poses up there).
  MVStereoFrontEnd node_;
  void eventsCallback(const std::vector<esvo::Event>& events, bool left) { if (node_.eventsCallback(events, left)) resetMap(); }
  void timeSurfaceCallback(int64_t stamp_ns, const uint8_t* ts_left, const uint8_t* ts_right) {
    if (node_.timeSurfaceCallback(stamp_ns, ts_left, ts_right)) resetMap();
  }
  void stampedPoseCallback(int64_t stamp_ns, const esvo::Pose& T_world_dvs) { if (node_.stampedPoseCallback(stamp_ns, T_world_dvs)) resetMap(); }
  bool getPoseAt(int64_t t_ns, esvo::Pose& T) const { return node_.getPoseAt(t_ns, T); }
  // dataTransferring (:552-668) into the inputs above; BM modes get the window events undenoised (see MappingLoopOnce)
  bool dataTransferring() {
    const bool ok = node_.dataTransferring();
    takeInputs(node_.vCloseEventsPtr_left_);
    return ok;
  }
  // What one pass of MappingLoop did.  gated: TS_history_.size() >= 10; transferred: dataTransferring's result; ran:
  // MappingAtTime was called (an observation was loaded -- publishKFPose then published stamp / T_world_kf); ok: it
  // reached the accumulation / fusion; published: publishPointCloud published `cloud` (world frame, f32 x,y,z).
  struct LoopResult {
    bool gated = false, transferred = false, ran = false, ok = false, published = false;
    int64_t stamp = 0; esvo::Pose T_world_kf{};
    size_t n_left = 0, n_right = 0, n_sgm = 0, n_window = 0, n_close = 0, n_st = 0, n_matches = 0;
    std::vector<float> cloud;
  };
  // one pass of MappingLoop's body (:196-225) with publishMappingResults / publishPointCloud (:960-1039) run in line
  bool MappingLoopOnce(LoopResult& res) {
    res = LoopResult();
    MVStereoFrontEnd::Pass p;
    const bool due = node_.prepare(p);
    res.gated = p.gated; res.transferred = p.transferred;
    if (!due) return false;
    takeInputs(node_.vDenoisedEventsPtr_left_);
    res.stamp = TS_obs_.first; res.T_world_kf = TS_obs_.second.tr_;                        // publishKFPose (:1041-1055)
    res.n_left = vEventsPtr_left_.size(); res.n_right = vEventsPtr_right_.size(); res.n_sgm = vEventsPtr_left_SGM_.size();
    res.n_window = node_.vALLEventsPtr_left_.size(); res.n_close = vCloseEventsPtr_left_.size(); res.n_st = st_map_.size();
    res.ran = true;
    res.ok = MappingAtTime();
    res.n_matches = vEMP_.size();
    if (res.ok) publishMappingResults(res);
    return res.ok;
  }
  // The map of the current DepthFrame: empty when none has been filled since it was made (a MappingAtTime that returned
  // before the accumulation, or a reset).
  void getMap(std::vector<esvo::DepthPoint>& out) {
    if (!depthFramePtr_ || depthFramePtr_->fresh_) { out.clear(); return; }
    getElements(out);
  }
  eMVStereoMode msm_;
  double EM_Slice_Thickness_ = 1e-3, EM_Time_THRESHOLD_ = 5e-5, EM_EPIPOLAR_THRESHOLD_ = 0.5, EM_TS_NCC_THRESHOLD_ = 0.1;   // :81-84
  size_t num_disparities_ = 16 * 3, block_size_ = 11, P1_ = 8 * 11 * 11, P2_ = 32 * 11 * 11;                                // :100-107
  size_t maxNumFusionFrames_ = 20, maxNumFusionPoints_ = 2000;
 private:
  void takeInputs(const std::vector<esvo::Event*>& bm_events) {
    TS_obs_ = node_.TS_obs_;
    vEventsPtr_left_ = node_.vEventsPtr_left_; vEventsPtr_right_ = node_.vEventsPtr_right_;
    t_lowBound_ = node_.t_lowBound_; t_upBound_ = node_.t_upBound_;
    vEventsPtr_left_SGM_ = node_.vEventsPtr_left_SGM_;
    vCloseEventsPtr_left_ = bm_events;
    st_map_ = node_.st_map_;
  }
  void resetMap() {
    dqvDepthPoints_.clear();
    esvo_mapping_reset(cs_->ctx());
    if (depthFramePtr_) depthFramePtr_->fresh_ = true;   // depthFramePtr_->clear()
  }
  // publishMappingResults -> publishPointCloud (:960-1039): the DepthMap at the frame's pose, nothing when it is empty
  void publishMappingResults(LoopResult& res) {
    std::vector<esvo::DepthPoint> elems;
    getMap(elems);
    frontend::packPointCloud(elems, depthFramePtr_->T_world_frame_, res.cloud);
    res.published = !res.cloud.empty();
  }
  // accumulation of modes 0, 1, 4 (:280-286,355-361,423-427): window of maxNumFusionFrames_ vectors, newest first, nearest wins
  bool accumulateNaive(std::vector<esvo::DepthPoint>& vdp) {
    dqvDepthPoints_.push_back(vdp);
    while (dqvDepthPoints_.size() > maxNumFusionFrames_) dqvDepthPoints_.pop_front();
    for (auto it = dqvDepthPoints_.rbegin(); it != dqvDepthPoints_.rend(); ++it) dFusor_.naive_propagation(*it, depthFramePtr_);
    return true;
  }
  // the PURE_SEMI_GLOBAL_MATCHING branch between the SGM call and the accumulation (:320-352) with createEdgeMask
  // (undistorted events, radius 0, :1130-1175) inlined: one Gaussian point per event whose rectified pixel lies right of
  // numDisparities and carries a non-negative disparity
  void sgmPoints(const std::vector<int16_t>& dispMap, std::vector<esvo::DepthPoint>& vdp_sgm) {
    const int W = cs_->width_, H = cs_->height_;
    if (lut_.empty()) { lut_.resize((size_t)2 * W * H); esvo_get_rectify_tables(cs_->ctx(), 0, nullptr, nullptr, lut_.data(), nullptr); }
    double d[4]; esvo_get_derived(cs_->ctx(), d);
    std::vector<esvo::EventMatchPair> pseudo;
    for (auto* e : vEventsPtr_left_SGM_) {
      const double* coor = &lut_[2 * ((size_t)e->y * W + e->x)];
      const int x = (int)std::floor(coor[0]), y = (int)std::floor(coor[1]);
      if (x < 0 || x >= W || y < 0 || y >= H) continue;
      if ((size_t)x < num_disparities_) continue;
      const double disp = dispMap[(size_t)y * W + x] / 16.0;
      if (disp < 0) continue;
      esvo::EventMatchPair s{};
      s.x_left[0] = x * 1.0; s.x_left[1] = y * 1.0;
      s.inv_depth = disp / (cs_->P_left_[0] * d[0]);
      s.cost = 0.0;
      std::copy(TS_obs_.second.tr_.begin(), TS_obs_.second.tr_.end(), s.T_world_virtual);
      pseudo.push_back(s);
    }
    vEMP2vDP(pseudo, vdp_sgm);
    for (size_t i = 0; i < vdp_sgm.size(); ++i) {       // DepthPoint dp(x, y): the reference passes (x, y) as (row, col) (:336)
      vdp_sgm[i].row = (int32_t)pseudo[i].x_left[0]; vdp_sgm[i].col = (int32_t)pseudo[i].x_left[1];
    }
  }
  core::EventMatcher em_;
  core::EventBM ebm_;
  core::DepthProblemSolver dpSolver_;
  core::DepthFusion dFusor_;
  core::DepthRegularization dRegularizor_;
  esvo::CameraSystem::Ptr cs_;
  core::DepthFrame::Ptr depthFramePtr_;
  PoseProvider getPoseAt_;
  std::vector<double> lut_;
};

// esvo_core::esvo_Tracking (esvo_Tracking.h:51-53; esvo_Tracking.cpp:79-265 TrackingLoop / refDataTransferring /
// curDataTransferring, :279-377 callbacks) without ROS.  The subscriptions become plain methods that fill the same buffers
// (refPCMap_, TS_history_, events_left_); the tf look-up becomes a pose provider; one pass of TrackingLoop's body is
// TrackingLoopOnce().  The registration itself runs on the device through RegProblemSolverLM (esvo_track_reset/solve).
class esvo_Tracking {
 public:
  enum TrackingStatus { IDLE, WORKING };
  using PoseProvider = std::function<bool(int64_t /*stamp ns*/, esvo::Pose& /*T_world_dvs*/)>;   // getPoseAt (:359-377)
  esvo_Tracking(esvo::CameraSystem::Ptr cs, core::RegProblemType rpType = core::REG_ANALYTICAL, size_t TS_HISTORY_LENGTH = 100,
                size_t REF_HISTORY_LENGTH = 5)
      : rpSolver_(cs, rpType), cs_(cs), rpType_(rpType), TS_HISTORY_LENGTH_(TS_HISTORY_LENGTH), REF_HISTORY_LENGTH_(REF_HISTORY_LENGTH) {
    T_world_cur_ = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  }
  void setPoseProvider(PoseProvider f) { getPoseAt_ = std::move(f); }
  // ---- callbacks (:279-357) ----
  // refMapCallback: the local map as the mapping node publishes it (pcl::PointXYZ: f32 x,y,z in the WORLD frame, i.e. the
  // output of frontend::packPointCloud); at most REF_HISTORY_LENGTH maps are kept.
  void refMapCallback(int64_t stamp_ns, const std::vector<float>& xyz) {
    refPCMap_[stamp_ns] = RefMap{std::make_shared<std::vector<float>>(xyz), xyz.size() / 3};
    while (refPCMap_.size() > REF_HISTORY_LENGTH_) refPCMap_.erase(refPCMap_.begin());
  }
  // Device form: the cloud of n_points the mapper published on this context at stamp_ns (esvo_map_publish_dev); it stays
  // there, and refDataTransferring adopts it (esvo_track_adopt_map_dev).
  void refMapCallback(int64_t stamp_ns, size_t n_points) {
    refPCMap_[stamp_ns] = RefMap{nullptr, n_points};
    while (refPCMap_.size() > REF_HISTORY_LENGTH_) refPCMap_.erase(refPCMap_.begin());
  }
  // timeSurfaceCallback: mono8 left image (H*W); the tracker only reads the left one (:331-349).
  void timeSurfaceCallback(int64_t stamp_ns, const uint8_t* time_surface_left) {
    const size_t n = (size_t)cs_->width_ * cs_->height_;
    TS_history_[stamp_ns] = TsEntry{std::vector<uint8_t>(time_surface_left, time_surface_left + n), TS_id_++};
    while (TS_history_.size() > TS_HISTORY_LENGTH_) TS_history_.erase(TS_history_.begin());
  }
  // Device form: the left image just built on this context at stamp_ns; the history keeps the stamp, and the registration
  // reads the newest camera-0 build (esvo_track_reset with ts_left = NULL).
  void timeSurfaceCallback(int64_t stamp_ns) {
    TS_history_[stamp_ns] = TsEntry{{}, TS_id_++};
    while (TS_history_.size() > TS_HISTORY_LENGTH_) TS_history_.erase(TS_history_.begin());
  }
  // eventsCallback: insertion-sorted event buffer, capped at 5e6 (:294-321)
  void eventsCallback(const std::vector<esvo::Event>& events) { frontend::queueEvents(events_left_, events, MAX_EVENT_QUEUE_LENGTH); }
  static constexpr size_t MAX_EVENT_QUEUE_LENGTH = 5000000;
  // Device form: the left events are in camera 0's time-surface log on this context, total_left of them since it was reset
  // (esvo_time_surface::TimeSurface::eventsPushed).  events_left_ stays empty; curDataTransferring counts on the device
  // (esvo_events_lower_bound_dev over the deque's place in the log, [max(push index at the last reset(), total - 5e6), total)).
  void eventsCallback(size_t total_left) { log_total_ = total_left; events_in_log_ = true; }
  // ---- refDataTransferring (:177-211) ----
  bool refDataTransferring() {
    ref_.t_ = refPCMap_.rbegin()->first;
    if (ESVO_System_Status_ == "INITIALIZATION" && ets_ == IDLE) ref_.tr_ = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    if (ESVO_System_Status_ == "WORKING" || (ESVO_System_Status_ == "INITIALIZATION" && ets_ == WORKING)) {
      if (!getPoseAt_ || !getPoseAt_(ref_.t_, ref_.tr_)) return false;   // the reference exit(-1)s here ("logic error")
    }
    const RefMap& m = refPCMap_.rbegin()->second;
    ref_.on_device_ = !m.host;
    if (m.host) ref_.vPointXYZ_ = *m.host;             // the reference keeps pointers into the cloud; the device path permutes a copy
    else {
      ref_.vPointXYZ_.clear();
      if (esvo_track_adopt_map_dev(cs_->ctx(), ref_.t_, nullptr) != ESVO_OK) { error_ = std::string("adopting the map: ") + esvo_last_error(cs_->ctx()); return false; }
    }
    return true;
  }
  // ---- curDataTransferring (:213-245) ----
  bool curDataTransferring() {
    const int64_t t_last = cur_.t_;
    auto TS_it = TS_history_.rbegin();
    if (cur_.t_ == TS_it->first) return false;        // TS_history may not have been updated yet
    cur_.t_ = TS_it->first;
    cur_.ts_left = TS_it->second.left.empty() ? nullptr : TS_it->second.left.data();   // empty: the newest camera-0 build
    if (ESVO_System_Status_ == "INITIALIZATION" && ets_ == IDLE) cur_.tr_ = ref_.tr_;
    if (ESVO_System_Status_ == "WORKING" || (ESVO_System_Status_ == "INITIALIZATION" && ets_ == WORKING)) cur_.tr_ = T_world_cur_;
    return numEventsBetween(t_last, cur_.t_, cur_.numEventsSinceLastObs_);
  }
  // ---- one pass of TrackingLoop's body (:84-171).  Returns true when a pose was produced (then also in T_world_cur_). ----
  bool TrackingLoopOnce() {
    if (refPCMap_.size() < 1 || TS_history_.size() < 1) return false;                       // keep idling
    if (ESVO_System_Status_ == "INITIALIZATION" && ets_ == WORKING) { reset(); return false; }
    if (ESVO_System_Status_ == "TERMINATE") return false;
    if (frontend::toSec(ref_.t_) < frontend::toSec(refPCMap_.rbegin()->first))            // new reference map arrived
      if (!refDataTransferring()) { if (error_.empty()) error_ = "no pose for the reference map"; return false; }
    if (frontend::toSec(cur_.t_) < frontend::toSec(TS_history_.rbegin()->first)) {          // new observation arrived
      if (frontend::toSec(ref_.t_) >= frontend::toSec(TS_history_.rbegin()->first)) {       // obs must come after the ref (reference: exit(-1))
        error_ = "time-surface observation is not newer than the reference map";
        return false;
      }
      if (!curDataTransferring()) return false;
    } else return false;
    if (rpSolver_.resetRegProblem(&ref_, &cur_)) {
      if (ets_ == IDLE) ets_ = WORKING;
      if (ESVO_System_Status_ != "WORKING") ESVO_System_Status_ = "WORKING";
      const bool ok = rpType_ == core::REG_NUMERICAL ? rpSolver_.solve_numerical() : rpSolver_.solve_analytical();
      if (!ok) { error_ = std::string("tracking solve: ") + esvo_last_error(cs_->ctx()); return false; }   // device / ABI error only
      T_world_cur_ = cur_.tr_;
      lTimestamp_.push_back(cur_.t_); lPose_.push_back(cur_.tr_);                             // publishPose / saveTrajectory payload
      return true;
    }
    ESVO_System_Status_ = "INITIALIZATION";
    ets_ = IDLE;
    return false;
  }
  void reset() { ets_ = IDLE; TS_id_ = 0; TS_history_.clear(); refPCMap_.clear(); events_left_.clear(); log_reset_ = log_total_; }   // (:247-255)
  // saveTrajectory (:430-462): per tracked frame "<std::to_string(t.toSec())> tx ty tz qx qy qz qw", fixed notation, precision 9
  // after the stamp; q = Eigen::Quaterniond(R) (esvo::quaternionFromRotation).  The translation is written as Eigen's default
  // IOFormat writes twc.transpose(): every column right-aligned to the widest of the three.  false if the file cannot be opened.
  bool saveTrajectory(const std::string& path) const {
    std::FILE* f = std::fopen(path.c_str(), "w");
    if (!f) return false;
    for (size_t i = 0; i < lPose_.size(); ++i) {
      const esvo::Pose& T = lPose_[i];
      const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
      double q[4];
      esvo::quaternionFromRotation(R, q);
      char t[3][64];
      int w = 0;
      for (int k = 0; k < 3; ++k) w = std::max(w, std::snprintf(t[k], sizeof(t[k]), "%.9f", T[4 * k + 3]));
      std::fprintf(f, "%s %*s %*s %*s %.9f %.9f %.9f %.9f\n", std::to_string(frontend::toSec(lTimestamp_[i])).c_str(), w, t[0], w, t[1], w, t[2],
                   q[0], q[1], q[2], q[3]);
    }
    return std::fclose(f) == 0;
  }

  std::string ESVO_System_Status_ = "INITIALIZATION";   // the /ESVO_SYSTEM_STATUS parameter
  std::string error_;                                  // set where the reference exit(-1)s; the pass then returned false
  TrackingStatus ets_ = IDLE;
  core::RefFrame ref_;
  core::CurFrame cur_;
  esvo::Pose T_world_cur_;
  std::vector<int64_t> lTimestamp_;
  std::vector<esvo::Pose> lPose_;
  core::RegProblemSolverLM rpSolver_;
 private:
  // numEventsSinceLastObs_ (:240-263): lower_bound(t_cur) - lower_bound(t_last) + 1.  The reference only logs it
  // (RegProblemSolverLM.cpp:47-51).  In the device form, a bound that lies among events folded out of the resident log cannot be
  // answered (ESVO_ERR_UNSUPPORTED); the count is then SIZE_MAX ("unknown") and tracking goes on.  Any other failure (a device
  // error, unordered input, a front past the log) sets error_ and returns false, which stops the pass.
  bool numEventsBetween(int64_t t_last, int64_t t_cur, size_t& count) {
    if (!events_in_log_) { count = frontend::lowerBound(events_left_, t_cur) - frontend::lowerBound(events_left_, t_last) + 1; return true; }
    const size_t lo = log_total_ > MAX_EVENT_QUEUE_LENGTH ? log_total_ - MAX_EVENT_QUEUE_LENGTH : 0;
    const int64_t front = (int64_t)std::max(log_reset_, lo), q[2] = {t_last, t_cur};
    int64_t idx[2] = {-2, -2};
    const int rc = esvo_events_lower_bound_dev(cs_->ctx(), 0, front, q, 2, idx);
    if (rc == ESVO_OK) { count = (size_t)(idx[1] - idx[0]) + 1; return true; }
    if (rc == ESVO_ERR_UNSUPPORTED && (idx[0] == -1 || idx[1] == -1)) { count = SIZE_MAX; return true; }   // folded out
    error_ = std::string("event count: ") + esvo_last_error(cs_->ctx());
    return false;
  }
  struct TsEntry { std::vector<uint8_t> left; size_t id; };
  esvo::CameraSystem::Ptr cs_;
  core::RegProblemType rpType_;
  size_t TS_HISTORY_LENGTH_, REF_HISTORY_LENGTH_, TS_id_ = 0;
  struct RefMap { std::shared_ptr<std::vector<float>> host; size_t n; };   // host == nullptr: published on the device
  std::map<int64_t, RefMap> refPCMap_;
  std::map<int64_t, TsEntry> TS_history_;
  std::deque<esvo::Event> events_left_;
  size_t log_total_ = 0, log_reset_ = 0;   // device form: left events in the log; how many there were at the last reset()
  bool events_in_log_ = false;
  PoseProvider getPoseAt_;
};
}  // namespace esvo_core
