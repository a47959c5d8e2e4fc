// esvo_b200 -- recorded ROS1 bags without ROS: the dvs_msgs/EventArray and sensor_msgs/CameraInfo topics of a bag, read
// from a memory-mapped file.  Header-only, host code, no ROS and no compression library.
//
// Format: ROS bag 2.0 (http://wiki.ros.org/Bags/Format/2.0).  After the "#ROSBAG V2.0\n" line the file is a sequence of
// records, each  u32 header_len | header | u32 data_len | data,  the header a sequence of  u32 len | "name=value"  fields,
// "op" naming the record type.  The records are scanned in file order:
//   0x03 bag header            -- checked, nothing else is needed from it;
//   0x05 chunk                 -- compression=none: its data is again a sequence of records, scanned in place; bz2 / lz4
//                                 are refused by RosBag(path); RosBag(path, inflate_device) inflates them first, on the
//                                 device (include/esvo_b200_inflate.h: no decompression library), and scans the inflated
//                                 bytes;
//   0x07 connection            -- conn id -> topic and type (inside chunks and in the index section; either suffices);
//   0x02 message data          -- conn id, receipt time, the serialised message, used where it lies in the map;
//   0x04 index data, 0x06 chunk info -- skipped.
// Every failure (unsupported version, compressed chunk, truncated file, wrong topic type) throws std::runtime_error with
// the reason; nothing is read outside the mapped file.
//
// dvs_msgs/EventArray:  Header header | u32 height | u32 width | Event[] events  (u32 count, then count * 13 bytes);
// dvs_msgs/Event:       u16 x | u16 y | time ts (u32 sec, u32 nsec) | bool polarity -- exactly the records
//                       esvo_ts_push_event_array takes, so the events go to the device as they lie in the file.
// sensor_msgs/CameraInfo: Header | u32 height | u32 width | string distortion_model | f64[] D | f64[9] K | f64[9] R |
//                       f64[12] P | binning, roi (unused).
#pragma once
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cstdint>
#include <cstring>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "esvo_core.hpp"

namespace esvo {

// The inflating reader found compressed chunks but could not get a CUDA device to inflate them on.
struct InflateDeviceError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

class RosBag {
 public:
  struct Message { uint32_t conn; uint64_t time; const uint8_t* data; size_t size; };
  struct Connection { std::string topic, type; };

  // Host only: a bag with a compressed chunk is refused.
  explicit RosBag(const std::string& path) {
    map(path);
    try { scan(); } catch (...) { unmap(); throw; }
  }
  // Inflating: the bz2 and lz4 chunks are inflated on device inflate_device (an inflater with `scratch` bytes of device
  // memory, created only if the bag has such a chunk) in one esvo_inflate_chunks call, into host memory the RosBag owns
  // for its lifetime; the messages of those chunks point there.  This costs host memory equal to the uncompressed chunks.
  // A bag without compressed chunks is read as RosBag(path) reads it.
  RosBag(const std::string& path, int inflate_device, size_t scratch = size_t(1) << 30) {
    map(path);
    try { inflate(inflate_device, scratch); scan(); } catch (...) { unmap(); throw; }
  }
  ~RosBag() { unmap(); }
  RosBag(const RosBag&) = delete;
  RosBag& operator=(const RosBag&) = delete;

  // bytes of inflated chunk data the bag holds (0 without compressed chunks)
  size_t inflatedBytes() const { return inflated_.size(); }

  const std::map<uint32_t, Connection>& connections() const { return conns_; }
  // the type of a topic ("" if the bag has no connection on it)
  std::string topicType(const std::string& topic) const {
    for (const auto& c : conns_) if (c.second.topic == topic) return c.second.type;
    return "";
  }
  // the messages of one topic in file order; throws if the topic is missing or of another type than `type`
  std::vector<const Message*> messages(const std::string& topic, const std::string& type) const {
    const std::string have = topicType(topic);
    if (have.empty()) throw std::runtime_error("rosbag: no topic " + topic);
    if (have != type) throw std::runtime_error("rosbag: topic " + topic + " is " + have + ", not " + type);
    std::vector<const Message*> out;
    for (const auto& m : msgs_) {
      auto it = conns_.find(m.conn);
      if (it != conns_.end() && it->second.topic == topic) out.push_back(&m);
    }
    return out;
  }

 private:
  using Fields = std::map<std::string, std::pair<const uint8_t*, size_t>>;
  static uint32_t u32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
  static uint64_t u64(const uint8_t* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
  [[noreturn]] static void truncated() { throw std::runtime_error("rosbag: truncated file"); }

  void map(const std::string& path) {
    const int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) throw std::runtime_error("rosbag: cannot open " + path);
    struct stat st {};
    if (::fstat(fd, &st) != 0) { ::close(fd); throw std::runtime_error("rosbag: cannot stat " + path); }
    size_ = (size_t)st.st_size;
    if (size_) {
      void* m = ::mmap(nullptr, size_, PROT_READ, MAP_PRIVATE, fd, 0);
      ::close(fd);
      if (m == MAP_FAILED) throw std::runtime_error("rosbag: cannot map " + path);
      base_ = (const uint8_t*)m;
    } else {
      ::close(fd);
    }
  }
  void unmap() { if (base_) ::munmap((void*)base_, size_); base_ = nullptr; }

  static Fields fields(const uint8_t* p, size_t n) {
    Fields f;
    size_t o = 0;
    while (o < n) {
      if (n - o < 4) truncated();
      const uint32_t len = u32(p + o); o += 4;
      if (len > n - o) truncated();
      const uint8_t* e = (const uint8_t*)std::memchr(p + o, '=', len);
      if (!e) throw std::runtime_error("rosbag: malformed record header");
      f[std::string((const char*)p + o, (size_t)(e - (p + o)))] = {e + 1, (size_t)(p + o + len - (e + 1))};
      o += len;
    }
    return f;
  }
  static const std::pair<const uint8_t*, size_t>& field(const Fields& f, const char* name, size_t min_size) {
    auto it = f.find(name);
    if (it == f.end() || it->second.second < min_size) throw std::runtime_error(std::string("rosbag: record without ") + name);
    return it->second;
  }
  static std::string str(const std::pair<const uint8_t*, size_t>& v) { return std::string((const char*)v.first, v.second); }

  // the records in [p, p + n); in_chunk: records of an uncompressed chunk's data
  void records(const uint8_t* p, size_t n, bool in_chunk) {
    size_t o = 0;
    while (o < n) {
      if (n - o < 4) truncated();
      const uint32_t hl = u32(p + o); o += 4;
      if (hl > n - o) truncated();
      const Fields f = fields(p + o, hl); o += hl;
      if (n - o < 4) truncated();
      const uint32_t dl = u32(p + o); o += 4;
      if (dl > n - o) truncated();
      const uint8_t* data = p + o; o += dl;
      const auto& op = field(f, "op", 1);
      switch (op.first[0]) {
        case 0x03:
          if (in_chunk || have_header_) throw std::runtime_error("rosbag: misplaced bag header");
          have_header_ = true;
          index_pos_ = u64(field(f, "index_pos", 8).first);
          chunk_count_ = u32(field(f, "chunk_count", 4).first);
          break;
        case 0x05: {
          if (in_chunk) throw std::runtime_error("rosbag: chunk inside a chunk");
          ++chunks_;
          const std::string comp = str(field(f, "compression", 0));
          const auto inf = inflated_at_.find(data);
          if (inf != inflated_at_.end()) {
            records(inflated_.data() + inf->second.first, inf->second.second, true);
            break;
          }
          if (comp != "none" && inflating_)
            throw std::runtime_error("rosbag: chunk compression '" + comp + "' is not supported (none, bz2 and lz4 are)");
          if (comp != "none")
            throw std::runtime_error("rosbag decompress: chunk compression '" + comp +
                                     "' is not supported (only uncompressed bags; `rosbag decompress` the file first)");
          records(data, dl, true);
          break;
        }
        case 0x07: {
          const uint32_t id = u32(field(f, "conn", 4).first);
          const Fields cf = fields(data, dl);
          conns_[id] = Connection{str(field(f, "topic", 0)), str(field(cf, "type", 0))};
          break;
        }
        case 0x02: {
          if (!in_chunk) throw std::runtime_error("rosbag: message data outside a chunk");
          msgs_.push_back(Message{u32(field(f, "conn", 4).first), u64(field(f, "time", 8).first), data, dl});
          break;
        }
        case 0x04: case 0x06: break;
        default: throw std::runtime_error("rosbag: unknown record op " + std::to_string((int)op.first[0]));
      }
    }
  }
  void checkMagic() const {
    static const char magic[] = "#ROSBAG V2.0\n";
    if (size_ >= 9 && std::memcmp(base_, "#ROSBAG V", 9) == 0 && (size_ < 13 || std::memcmp(base_, magic, 13) != 0)) {
      size_t e = 9;
      while (e < size_ && e < 16 && base_[e] != '\n') ++e;
      throw std::runtime_error("rosbag: unsupported bag version V" + std::string((const char*)base_ + 9, e - 9) + " (only 2.0)");
    }
    if (size_ < 13 || std::memcmp(base_, magic, 13) != 0) throw std::runtime_error("rosbag: not a ROS bag");
  }
  void scan() {
    checkMagic();
    records(base_ + 13, size_ - 13, false);
    // a file cut at a record boundary: the bag header, chunks or the index section are missing
    if (!have_header_ || chunks_ < chunk_count_ || index_pos_ > size_) truncated();
  }

  // Walks the top-level records, collects the bz2 / lz4 chunks (their header's `size` is required) and inflates them all
  // in one call.
  void inflate(int device, size_t scratch) {
    inflating_ = true;
    checkMagic();
    std::vector<esvo_chunk> cs;
    std::vector<size_t> at;   // file offset of each chunk record
    size_t o = 13, total = 0;
    while (o < size_) {
      const size_t rec = o;
      if (size_ - o < 4) truncated();
      const uint32_t hl = u32(base_ + o); o += 4;
      if (hl > size_ - o) truncated();
      const Fields f = fields(base_ + o, hl); o += hl;
      if (size_ - o < 4) truncated();
      const uint32_t dl = u32(base_ + o); o += 4;
      if (dl > size_ - o) truncated();
      const uint8_t* data = base_ + o; o += dl;
      if (field(f, "op", 1).first[0] != 0x05) continue;
      const std::string comp = str(field(f, "compression", 0));
      if (comp != "bz2" && comp != "lz4") continue;
      esvo_chunk c{};
      c.src = data; c.src_size = dl;
      c.dst_size = u32(field(f, "size", 4).first);
      c.codec = comp == "bz2" ? ESVO_CODEC_BZ2 : ESVO_CODEC_LZ4;
      cs.push_back(c); at.push_back(rec);
      total += c.dst_size;
    }
    if (cs.empty()) return;
    inflated_.resize(total);
    size_t off = 0;
    for (esvo_chunk& c : cs) {
      c.dst = inflated_.data() + off;
      inflated_at_[c.src] = {off, (size_t)c.dst_size};
      off += c.dst_size;
    }
    esvo_inflater* inf = nullptr;
    const int rc = esvo_inflater_create(device, scratch, &inf);
    if (rc == ESVO_ERR_NO_DEVICE)
      throw InflateDeviceError("rosbag: the bag has compressed chunks and there is no CUDA device " + std::to_string(device) +
                               " to inflate them on (no CPU fallback)");
    if (rc != ESVO_OK) throw InflateDeviceError("rosbag: cannot create an inflater on device " + std::to_string(device));
    const int r = esvo_inflate_chunks(inf, cs.data(), (int)cs.size());
    std::string why = esvo_inflater_last_error(inf);
    esvo_inflater_destroy(inf);
    if (r == ESVO_OK) return;
    const size_t colon = why.find(": ");
    if (why.compare(0, 6, "chunk ") == 0 && colon != std::string::npos) why = why.substr(colon + 2);   // the reason alone
    for (size_t k = 0; k < cs.size(); ++k)
      if (cs[k].status != ESVO_OK)
        throw std::runtime_error("rosbag: compressed chunk at file offset " + std::to_string(at[k]) + " refused: " + why);
    throw std::runtime_error("rosbag: inflating the compressed chunks failed: " + why);
  }

  const uint8_t* base_ = nullptr;
  size_t size_ = 0;
  bool inflating_ = false;
  std::vector<uint8_t> inflated_;                                        // the inflated chunks, in file order
  std::map<const uint8_t*, std::pair<size_t, size_t>> inflated_at_;    // chunk data in the map -> (offset, size) in inflated_
  bool have_header_ = false;
  uint64_t index_pos_ = 0;
  uint32_t chunk_count_ = 0, chunks_ = 0;
  std::map<uint32_t, Connection> conns_;
  std::vector<Message> msgs_;
};

namespace detail {
struct Reader {   // bounds-checked little-endian reads over one serialised message
  const uint8_t* p; size_t n, o = 0;
  void need(size_t k) { if (k > n - o) throw std::runtime_error("rosbag: truncated message"); }
  uint32_t u32() { need(4); uint32_t v; std::memcpy(&v, p + o, 4); o += 4; return v; }
  double f64() { need(8); double v; std::memcpy(&v, p + o, 8); o += 8; return v; }
  std::string str() { const uint32_t k = u32(); need(k); std::string s((const char*)p + o, k); o += k; return s; }
  void header() { u32(); u32(); u32(); str(); }   // std_msgs/Header: seq, stamp, frame_id
};
inline int64_t wireStamp(const uint8_t* r) {      // ros::Time::toNSec of a wire record's ts
  uint32_t sec, nsec;
  std::memcpy(&sec, r + 4, 4); std::memcpy(&nsec, r + 8, 4);
  return (int64_t)sec * 1000000000LL + (int64_t)nsec;
}
}  // namespace detail

constexpr size_t kEventWireBytes = 13;

// sensor_msgs/CameraInfo -> esvo_calib (the first message of the topic).  plumb_bob takes D = (k1, k2, p1, p2) and an
// optional fifth coefficient k3 that must be 0 (esvo_calib has four); equidistant takes D = (k1, k2, k3, k4).
inline esvo_calib cameraInfoCalib(const RosBag& bag, const std::string& topic) {
  const auto ms = bag.messages(topic, "sensor_msgs/CameraInfo");
  if (ms.empty()) throw std::runtime_error("rosbag: no message on " + topic);
  detail::Reader r{ms[0]->data, ms[0]->size};
  r.header();
  esvo_calib c{};
  c.height = (int32_t)r.u32(); c.width = (int32_t)r.u32();
  const std::string model = r.str();
  if (model == "plumb_bob") c.distortion_model = ESVO_DIST_PLUMB_BOB;
  else if (model == "equidistant") c.distortion_model = ESVO_DIST_EQUIDISTANT;
  else throw std::runtime_error("rosbag: " + topic + ": distortion model '" + model + "' is not supported");
  const uint32_t nd = r.u32();
  if (nd < 4 || nd > 5 || (nd == 5 && c.distortion_model != ESVO_DIST_PLUMB_BOB))
    throw std::runtime_error("rosbag: " + topic + ": " + std::to_string(nd) + " distortion coefficients for " + model);
  for (int i = 0; i < 4; ++i) c.D[i] = r.f64();
  if (nd == 5 && r.f64() != 0.0) throw std::runtime_error("rosbag: " + topic + ": plumb_bob k3 != 0 is not supported");
  for (double& v : c.K) v = r.f64();
  for (double& v : c.R) v = r.f64();
  for (double& v : c.P) v = r.f64();
  return c;
}

// A cursor over one dvs_msgs/EventArray topic.  takeBefore(t) hands out, as runs into the mapped file, every event not
// handed out yet whose stamp is < t -- the events of one sync tick.  Event stamps must not decrease along the topic; a
// message is split by a binary search over its records, and messages without events are stepped over.
class RosBagEvents {
 public:
  RosBagEvents(const RosBag& bag, const std::string& topic) {
    for (const RosBag::Message* m : bag.messages(topic, "dvs_msgs/EventArray")) {
      detail::Reader r{m->data, m->size};
      r.header(); r.u32(); r.u32();
      const uint32_t n = r.u32();
      if ((size_t)n * kEventWireBytes > r.n - r.o) throw std::runtime_error("rosbag: truncated message on " + topic);
      if (n) msgs_.push_back(EventRun{r.p + r.o, n});
      total_ += n;
    }
  }
  size_t total() const { return total_; }
  size_t taken() const { return taken_; }
  // every non-empty message's event block, in file order, whatever takeBefore has handed out (e.g. for a hot-pixel count
  // over the whole topic, esvo_hotpix_count_event_array)
  const std::vector<EventRun>& runs() const { return msgs_; }
  bool done() const { return k_ == msgs_.size(); }
  // stamp of the next event not handed out (undefined once done())
  int64_t nextStamp() const { return detail::wireStamp(msgs_[k_].data + pos_ * kEventWireBytes); }
  std::vector<EventRun> takeBefore(int64_t t_ns) {
    std::vector<EventRun> out;
    while (k_ < msgs_.size()) {
      const EventRun& m = msgs_[k_];
      size_t lo = pos_, hi = m.n;   // first record at or after pos_ with stamp >= t_ns
      while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (detail::wireStamp(m.data + mid * kEventWireBytes) < t_ns) lo = mid + 1; else hi = mid;
      }
      if (lo > pos_) { out.push_back(EventRun{m.data + pos_ * kEventWireBytes, lo - pos_}); taken_ += lo - pos_; }
      if (lo < m.n) { pos_ = lo; break; }
      ++k_; pos_ = 0;
    }
    return out;
  }

 private:
  std::vector<EventRun> msgs_;   // the non-empty messages' event blocks, in file order
  size_t k_ = 0, pos_ = 0, total_ = 0, taken_ = 0;
};

}  // namespace esvo
