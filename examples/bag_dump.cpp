// Reads a ROS1 bag with include/esvo_b200/rosbag_events.hpp and dumps what the closed loop would take from it (no GPU):
//   bag_dump events <bag> <topic> <out.bin>              every event of an EventArray topic:
//                                                        u64 n; n wire records (13 bytes); i64 stamp[n] (the reader's decode)
//   bag_dump take <bag> <topic> <queries.bin> <out.bin>  takeBefore(t) for each i64 t of queries.bin, in order:
//                                                        per query u64 runs, u64 events; then every handed-out record
//   bag_dump calib <bag> <topic> <out.bin>               a CameraInfo topic: esvo_calib, then esvo_compute_rectify_tables'
//                                                        map1, map2 (f32), lut (f64 x 2), mask (u8), H*W each
//   A leading `--inflate-device N` opens the bag with RosBag(path, N): its bz2 / lz4 chunks are inflated on CUDA device N
//   (include/esvo_b200_inflate.h).  Without it the bag is read on the host only and compressed chunks are refused.
// Exit codes: 0 done, 2 compressed chunks and no CUDA device to inflate them on, 3 the bag was refused (the reason is
// printed), 64 usage.
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <fstream>
#include <string>
#include <vector>

#include "esvo_b200/rosbag_events.hpp"

template <class T> static void wr(std::ofstream& o, const T* p, size_t n) { o.write((const char*)p, (std::streamsize)(n * sizeof(T))); }

int main(int argc, char** argv) {
  int inflate_device = -1;
  if (argc > 2 && std::string(argv[1]) == "--inflate-device") {
    inflate_device = std::atoi(argv[2]);
    argv += 2; argc -= 2;
  }
  const std::string mode = argc > 1 ? argv[1] : "";
  if (!((mode == "events" && argc == 5) || (mode == "take" && argc == 6) || (mode == "calib" && argc == 5))) {
    std::printf("usage: bag_dump [--inflate-device N] events|calib <bag> <topic> <out.bin> | "
                "bag_dump [--inflate-device N] take <bag> <topic> <queries.bin> <out.bin>\n");
    return 64;
  }
  try {
    std::unique_ptr<esvo::RosBag> owned = inflate_device < 0 ? std::make_unique<esvo::RosBag>(argv[2])
                                                             : std::make_unique<esvo::RosBag>(argv[2], inflate_device);
    const esvo::RosBag& bag = *owned;
    std::ofstream o(argv[argc - 1], std::ios::binary);
    if (mode == "calib") {
      const esvo_calib c = esvo::cameraInfoCalib(bag, argv[3]);
      const size_t n = (size_t)c.width * c.height;
      std::vector<float> m1(n), m2(n); std::vector<double> lut(2 * n); std::vector<uint8_t> mask(n);
      if (esvo_compute_rectify_tables(&c, m1.data(), m2.data(), lut.data(), mask.data()) != ESVO_OK) {
        std::printf("esvo_compute_rectify_tables failed\n");
        return 3;
      }
      wr(o, &c, 1); wr(o, m1.data(), n); wr(o, m2.data(), n); wr(o, lut.data(), 2 * n); wr(o, mask.data(), n);
      return 0;
    }
    esvo::RosBagEvents ev(bag, argv[3]);
    std::vector<esvo::EventRun> all;
    if (mode == "events") {
      all = ev.takeBefore(INT64_MAX);
      const uint64_t n = ev.taken();
      wr(o, &n, 1);
      for (const auto& r : all) wr(o, r.data, r.n * esvo::kEventWireBytes);
      for (const auto& r : all)
        for (size_t i = 0; i < r.n; ++i) { const int64_t t = esvo::detail::wireStamp(r.data + i * esvo::kEventWireBytes); wr(o, &t, 1); }
      return 0;
    }
    std::ifstream q(argv[4], std::ios::binary);
    int64_t t;
    while (q.read((char*)&t, 8)) {
      const auto runs = ev.takeBefore(t);
      uint64_t k[2] = {runs.size(), 0};
      for (const auto& r : runs) k[1] += r.n;
      wr(o, k, 2);
      all.insert(all.end(), runs.begin(), runs.end());
    }
    for (const auto& r : all) wr(o, r.data, r.n * esvo::kEventWireBytes);
  } catch (const esvo::InflateDeviceError& e) {
    std::printf("%s\n", e.what());
    return 2;
  } catch (const std::exception& e) {
    std::printf("%s\n", e.what());
    return 3;
  }
  return 0;
}
