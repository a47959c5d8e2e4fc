// The tracker's event count (esvo_Tracking::curDataTransferring, numEventsSinceLastObs_) in its host form (events_left_ fed by
// eventsCallback) and in its device form (lower bounds over camera 0's time-surface log), side by side on one event stream.
// usage: tracker_count_dump <in.bin> <out.bin>
// in:  i32 n_ticks; i64 tick stamps[n_ticks]; i32 reset flags[n_ticks] (1 = reset() both trackers after the tick);
//      i32 n; u16 x[n]; u16 y[n]; i64 t[n]   (time-ordered)
// out: per tick u64 host count, u64 device count (0 when curDataTransferring returned false; SIZE_MAX = not answerable)
#include <cstdio>
#include <cstring>
#include <fstream>

#include "esvo_b200/esvo_core.hpp"

template <class T> static bool rd(std::ifstream& f, T* p, size_t n) { f.read((char*)p, (std::streamsize)(n * sizeof(T))); return (bool)f; }

int main(int argc, char** argv) {
  if (argc < 3) { std::printf("usage: tracker_count_dump <in.bin> <out.bin>\n"); return 64; }
  std::ifstream f(argv[1], std::ios::binary);
  int32_t nt, n;
  if (!rd(f, &nt, 1)) return 65;
  std::vector<int64_t> ticks((size_t)nt); std::vector<int32_t> resets((size_t)nt);
  if (!rd(f, ticks.data(), ticks.size()) || !rd(f, resets.data(), resets.size()) || !rd(f, &n, 1)) return 65;
  std::vector<uint16_t> x((size_t)n), y((size_t)n); std::vector<int64_t> t((size_t)n);
  if (!rd(f, x.data(), x.size()) || !rd(f, y.data(), y.size()) || !rd(f, t.data(), t.size())) return 65;
  esvo_calib l{}, r{};
  l.width = r.width = 346; l.height = r.height = 260;
  const double K[9] = {200, 0, 173, 0, 200, 130, 0, 0, 1}, R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  const double Pl[12] = {200, 0, 173, 0, 0, 200, 130, 0, 0, 0, 1, 0};
  std::memcpy(l.K, K, 72); std::memcpy(l.R, R, 72); std::memcpy(l.P, Pl, 96);
  std::memcpy(r.K, K, 72); std::memcpy(r.R, R, 72); std::memcpy(r.P, Pl, 96); r.P[3] = -20;
  esvo_params p; esvo_default_params(&p);
  p.patch_size_x = 15; p.patch_size_y = 7;   // the mapping patch of the shipped yamls (the defaults are larger than the device path takes)
  esvo::CameraSystem::Ptr cs;
  try { cs = std::make_shared<esvo::CameraSystem>(l, r, p, 0); }
  catch (const std::exception& e) { std::printf("%s\n", e.what()); return 2; }
  esvo_time_surface::TimeSurface ts(cs, 0);
  esvo_core::esvo_Tracking host(cs), dev(cs);
  std::ofstream o(argv[2], std::ios::binary);
  size_t next = 0;
  std::vector<esvo::Event> batch;
  for (int k = 0; k < nt; ++k) {
    batch.clear();
    while (next < (size_t)n && t[next] < ticks[(size_t)k]) { batch.push_back({x[next], y[next], t[next], true}); ++next; }
    if (!batch.empty() && !ts.eventsCallback(batch)) { std::printf("push: %s\n", esvo_last_error(cs->ctx())); return 3; }
    host.eventsCallback(batch);
    dev.eventsCallback(ts.eventsPushed());
    uint64_t c[2];
    esvo_core::esvo_Tracking* tr[2] = {&host, &dev};
    for (int i = 0; i < 2; ++i) {
      tr[i]->timeSurfaceCallback(ticks[(size_t)k]);
      c[i] = tr[i]->curDataTransferring() ? (uint64_t)tr[i]->cur_.numEventsSinceLastObs_ : 0;
      if (resets[(size_t)k]) tr[i]->reset();
    }
    o.write((const char*)c, sizeof(c));
  }
  return 0;
}
