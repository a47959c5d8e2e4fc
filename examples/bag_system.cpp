// The closed stereo-odometry loop (include/esvo_b200/esvo_system.hpp) on a recorded ROS1 bag, without ROS: the rig comes
// from the two sensor_msgs/CameraInfo topics, the events from the two dvs_msgs/EventArray topics, and each tick's events go
// to the device as they lie in the memory-mapped bag (esvo::RosBagEvents::takeBefore -> esvo_ts_push_event_array).
// The bag is opened with RosBag(path, 0): bz2 and lz4 chunks (rosbag record -j / --lz4, rosbag compress) are inflated on
// device 0 before the first tick (include/esvo_b200_inflate.h); a bag without compressed chunks creates no inflater.
// Parameters: the hkust yamls (examples/system_common.hpp, as examples/system_loop.cpp).  Writes the result file,
// trajectory and calls file of system_loop.cpp.
// usage: bag_system <bag> <left events topic> <right events topic> <left camera_info topic> <right camera_info topic>
//                   <result.bin> <trajectory.txt> [--t0-ns T] [--dt-ns D] [--ticks N] [--mapping-every M]
//                   [--calls calls.txt] [--profile] [--hot-pixels K]
//   --t0-ns: first sync tick (default: the first left event's stamp + dt); --dt-ns: tick period (default 10 ms, 100 Hz);
//   --ticks: number of ticks (default: until every event of both topics has been delivered); --mapping-every: 5.
//   --hot-pixels K: before the first tick, count each events topic over the whole bag, select the hot pixels with k = K
//   (include/esvo_b200_hotpix.h; 5 is the usual choice) and drop their events from then on, as the offline hot-pixel tool
//   of the reference's data preparation does; prints the number of hot pixels per camera.
// Exit codes: 0 done, 2 no CUDA device (also: compressed chunks and no device to inflate them on), 3 the bag cannot be read
// (e.g. a compressed chunk is refused) or its hot pixels cannot be selected (the reason is printed), 64 usage.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "esvo_b200/esvo_system.hpp"
#include "esvo_b200/rosbag_events.hpp"
#include "system_common.hpp"

int main(int argc, char** argv) {
  if (argc < 8) {
    std::printf("usage: bag_system <bag> <left events> <right events> <left camera_info> <right camera_info> <result.bin> "
                "<trajectory.txt> [--t0-ns T] [--dt-ns D] [--ticks N] [--mapping-every M] [--calls calls.txt] [--profile] [--hot-pixels K]\n");
    return 64;
  }
  int64_t t0 = INT64_MIN, dt = 10000000, n_ticks = -1;
  int mapping_every = 5;
  double hot_k = -1;
  bool profile = false;
  const char* calls = nullptr;
  for (int i = 8; i < argc; ++i) {
    const std::string a = argv[i];
    const bool has = i + 1 < argc;
    if (a == "--t0-ns" && has) t0 = std::strtoll(argv[++i], nullptr, 10);
    else if (a == "--dt-ns" && has) dt = std::strtoll(argv[++i], nullptr, 10);
    else if (a == "--ticks" && has) n_ticks = std::strtoll(argv[++i], nullptr, 10);
    else if (a == "--mapping-every" && has) mapping_every = std::atoi(argv[++i]);
    else if (a == "--calls" && has) calls = argv[++i];
    else if (a == "--profile") profile = true;
    else if (a == "--hot-pixels" && has) {
      char* end = nullptr;
      hot_k = std::strtod(argv[++i], &end);
      if (*end || !(hot_k >= 0) || !std::isfinite(hot_k)) { std::printf("--hot-pixels takes a finite k >= 0\n"); return 64; }
    }
    else { std::printf("unknown argument %s\n", a.c_str()); return 64; }
  }
  if (dt <= 0 || mapping_every <= 0) { std::printf("--dt-ns and --mapping-every must be positive\n"); return 64; }

  std::unique_ptr<esvo::RosBag> bag;
  std::unique_ptr<esvo::RosBagEvents> ev[2];
  esvo_calib cal[2];
  try {
    const auto i0 = std::chrono::steady_clock::now();
    bag = std::make_unique<esvo::RosBag>(argv[1], 0);
    if (bag->inflatedBytes())
      std::printf("inflated %zu bytes of compressed chunks in %.3f ms\n", bag->inflatedBytes(),
                  std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - i0).count());
    for (int c = 0; c < 2; ++c) {
      ev[c] = std::make_unique<esvo::RosBagEvents>(*bag, argv[2 + c]);
      cal[c] = esvo::cameraInfoCalib(*bag, argv[4 + c]);
    }
  } catch (const esvo::InflateDeviceError& e) { std::printf("%s\n", e.what()); return 2; }
  catch (const std::exception& e) { std::printf("%s\n", e.what()); return 3; }
  if (t0 == INT64_MIN) t0 = (ev[0]->done() ? 0 : ev[0]->nextStamp()) + dt;

  esvo::CameraSystem::Ptr cs;
  try { cs = std::make_shared<esvo::CameraSystem>(cal[0], cal[1], esvo_examples::hkustParams(), 0); }
  catch (const std::exception& e) { std::printf("%s\n", e.what()); return 2; }
  if (profile) esvo_profile(cs->ctx(), 0xff);
  if (hot_k >= 0) {
    for (int c = 0; c < 2; ++c) {
      std::vector<const uint8_t*> ptr;
      std::vector<size_t> n;
      for (const esvo::EventRun& r : ev[c]->runs()) { ptr.push_back(r.data); n.push_back(r.n); }
      int64_t n_hot = 0;
      if (esvo_hotpix_count_event_array(cs->ctx(), c, ptr.data(), n.data(), (int)ptr.size()) != ESVO_OK ||
          esvo_hotpix_select(cs->ctx(), c, hot_k, &n_hot) != ESVO_OK) {
        std::printf("hot pixels: %s\n", esvo_last_error(cs->ctx()));
        return 3;
      }
      std::printf("hot pixels %s: %lld\n", c ? "right" : "left", (long long)n_hot);
    }
  }

  esvo_core::esvo_System::Config cfg;
  cfg.t0_ns = t0; cfg.dt_ns = dt; cfg.mapping_every = mapping_every;
  esvo_core::esvo_System sys(cs, cfg);
  const auto w0 = std::chrono::steady_clock::now();
  for (int64_t k = 0; n_ticks < 0 ? !(ev[0]->done() && ev[1]->done()) : k < n_ticks; ++k) {
    const int64_t t = sys.nextTick();   // every event with stamp < t_k not delivered yet, straight out of the mapped file
    if (!sys.SpinOnce(ev[0]->takeBefore(t), ev[1]->takeBefore(t))) break;
  }
  esvo_sync(cs->ctx());
  const double wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - w0).count();
  return esvo_examples::writeOutputs(sys, *cs, profile, wall_ms, argv[6], argv[7], calls);
}
