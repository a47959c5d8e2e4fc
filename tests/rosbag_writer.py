"""A ROS bag 2.0 writer for the tests, written from the format description (http://wiki.ros.org/Bags/Format/2.0) and the
message definitions (dvs_msgs/Event{,Array}, sensor_msgs/{CameraInfo,Imu,Image}, std_msgs/Header), not from the reader.

Layout written: the version line; the bag header record (op 0x03, padded to 4 096 bytes); chunks (op 0x05) of message data
records (op 0x02), each followed by one index data record (op 0x04) per connection in it; then the index section: one
connection record (op 0x07) per connection and one chunk info record (op 0x06) per chunk.  The bag header's index_pos points
at the index section.  Connection records are also written into the chunk that first uses the connection (as rosbag does)
unless conn_in_chunks=False, when the index section holds the only copy.

compression="bz2" compresses each chunk with the standard library's bz2.  "lz4" only names the compression (the data stays
uncompressed; there is no lz4 in the standard library) -- enough for a reader that must refuse it by name.
"""
import bz2
import struct

import numpy as np

# dvs_msgs/Event: uint16 x, uint16 y, time ts, bool polarity -- packed, little-endian
EVENT_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("sec", "<u4"), ("nsec", "<u4"), ("polarity", "u1")])

# (type, md5sum, message_definition); the reader does not check the md5 sums
TYPES = {
    "dvs_msgs/EventArray": ("5e8beee5a6c107e504c2e78903c224b8",
                            "Header header\nuint32 height\nuint32 width\nEvent[] events\n"
                            "================================================================================\n"
                            "MSG: dvs_msgs/Event\nuint16 x\nuint16 y\ntime ts\nbool polarity\n"),
    "sensor_msgs/CameraInfo": ("c9a58c1b0b154e0e6da7578cb991d214",
                               "Header header\nuint32 height\nuint32 width\nstring distortion_model\nfloat64[] D\n"
                               "float64[9] K\nfloat64[9] R\nfloat64[12] P\nuint32 binning_x\nuint32 binning_y\n"
                               "RegionOfInterest roi\n"),
    "sensor_msgs/Imu": ("6a62c6daae103f4ff57a132d6f95cec2",
                        "Header header\ngeometry_msgs/Quaternion orientation\nfloat64[9] orientation_covariance\n"
                        "geometry_msgs/Vector3 angular_velocity\nfloat64[9] angular_velocity_covariance\n"
                        "geometry_msgs/Vector3 linear_acceleration\nfloat64[9] linear_acceleration_covariance\n"),
    "sensor_msgs/Image": ("060021388200f6f0f447d0fcd9c64743",
                          "Header header\nuint32 height\nuint32 width\nstring encoding\nuint8 is_bigendian\nuint32 step\n"
                          "uint8[] data\n"),
}


def _time(t_ns):
    return struct.pack("<II", int(t_ns) // 1_000_000_000, int(t_ns) % 1_000_000_000)


def _string(s):
    b = s.encode() if isinstance(s, str) else bytes(s)
    return struct.pack("<I", len(b)) + b


def _header(seq, t_ns, frame_id="dvs"):
    return struct.pack("<I", seq) + _time(t_ns) + _string(frame_id)


def event_array(x, y, t_ns, pol, stamp_ns, width=346, height=260, seq=0):
    """A serialised dvs_msgs/EventArray; pol are the polarity bytes as written (a bool is 0 / 1 on the wire, any byte here)."""
    t = np.asarray(t_ns, np.int64)
    ev = np.empty(t.size, EVENT_DTYPE)
    ev["x"] = x; ev["y"] = y; ev["sec"] = t // 1_000_000_000; ev["nsec"] = t % 1_000_000_000; ev["polarity"] = pol
    return _header(seq, stamp_ns) + struct.pack("<III", height, width, t.size) + ev.tobytes()


def event_array_raw(records, stamp_ns, width=346, height=260, seq=0):
    """A serialised dvs_msgs/EventArray from EVENT_DTYPE records as given (e.g. nsec >= 1e9)."""
    records = np.ascontiguousarray(records, EVENT_DTYPE)
    return _header(seq, stamp_ns) + struct.pack("<III", height, width, records.size) + records.tobytes()


def camera_info(width, height, model, D, K, R, P, stamp_ns=0):
    return (_header(0, stamp_ns) + struct.pack("<II", height, width) + _string(model) +
            struct.pack("<I", len(D)) + np.asarray(D, "<f8").tobytes() + np.asarray(K, "<f8").tobytes() +
            np.asarray(R, "<f8").tobytes() + np.asarray(P, "<f8").tobytes() +
            struct.pack("<II", 0, 0) + struct.pack("<IIIIB", 0, 0, 0, 0, 0))


def imu(stamp_ns, seq=0):
    v = np.arange(4 + 9 + 3 + 9 + 3 + 9, dtype="<f8") * 0.25
    return _header(seq, stamp_ns, "imu") + v.tobytes()


def image(stamp_ns, width=34, height=26, seq=0):
    data = (np.arange(width * height) % 251).astype(np.uint8).tobytes()
    return _header(seq, stamp_ns, "cam") + struct.pack("<II", height, width) + _string("mono8") + struct.pack("<BI", 0, width) + _string(data)


def _fields(**kw):
    out = b""
    for k, v in kw.items():
        f = k.encode() + b"=" + v
        out += struct.pack("<I", len(f)) + f
    return out


def _record(header, data):
    return struct.pack("<I", len(header)) + header + struct.pack("<I", len(data)) + data


class BagWriter:
    def __init__(self, path, chunk_threshold=768 * 1024, compression="none", conn_in_chunks=True):
        self.path, self.threshold, self.compression, self.conn_in_chunks = path, chunk_threshold, compression, conn_in_chunks
        self.conns = {}            # topic -> (id, type)
        self.conn_written = set()
        self.out = bytearray(b"#ROSBAG V2.0\n")
        self.header_pos = len(self.out)
        self.out += b"\0" * 4096   # the bag header record, written at close
        self.chunk = bytearray()
        self.chunk_index = {}      # conn -> [(time, offset)]
        self.chunk_infos = []      # (chunk_pos, start, end, {conn: count})
        self.t_lo = self.t_hi = None

    def _conn_record(self, topic):
        cid, typ = self.conns[topic]
        md5, text = TYPES[typ]
        data = _fields(topic=topic.encode(), type=typ.encode(), md5sum=md5.encode(), message_definition=text.encode())
        return _record(_fields(op=b"\x07", conn=struct.pack("<I", cid), topic=topic.encode()), data)

    def write(self, topic, msgtype, t_ns, payload):
        if topic not in self.conns:
            self.conns[topic] = (len(self.conns), msgtype)
        cid, typ = self.conns[topic]
        assert typ == msgtype
        if self.conn_in_chunks and topic not in self.conn_written:
            self.chunk += self._conn_record(topic)
            self.conn_written.add(topic)
        self.chunk_index.setdefault(cid, []).append((int(t_ns), len(self.chunk)))
        self.chunk += _record(_fields(op=b"\x02", conn=struct.pack("<I", cid), time=_time(t_ns)), payload)
        self.t_lo = t_ns if self.t_lo is None else min(self.t_lo, t_ns)
        self.t_hi = t_ns if self.t_hi is None else max(self.t_hi, t_ns)
        if len(self.chunk) >= self.threshold:
            self._flush()

    def _flush(self):
        if not self.chunk:
            return
        raw = bytes(self.chunk)
        data = bz2.compress(raw) if self.compression == "bz2" else raw
        pos = len(self.out)
        self.out += _record(_fields(op=b"\x05", compression=self.compression.encode(), size=struct.pack("<I", len(raw))), data)
        counts = {}
        for cid, entries in sorted(self.chunk_index.items()):
            body = b"".join(_time(t) + struct.pack("<I", off) for t, off in entries)
            self.out += _record(_fields(op=b"\x04", ver=struct.pack("<I", 1), conn=struct.pack("<I", cid),
                                        count=struct.pack("<I", len(entries))), body)
            counts[cid] = len(entries)
        self.chunk_infos.append((pos, self.t_lo, self.t_hi, counts))
        self.chunk = bytearray(); self.chunk_index = {}; self.t_lo = self.t_hi = None

    def close(self):
        self._flush()
        index_pos = len(self.out)
        for topic in self.conns:
            self.out += self._conn_record(topic)
        for pos, lo, hi, counts in self.chunk_infos:
            body = b"".join(struct.pack("<II", c, n) for c, n in counts.items())
            self.out += _record(_fields(op=b"\x06", ver=struct.pack("<I", 1), chunk_pos=struct.pack("<Q", pos), start_time=_time(lo),
                                        end_time=_time(hi), count=struct.pack("<I", len(counts))), body)
        hdr = _fields(op=b"\x03", index_pos=struct.pack("<Q", index_pos), conn_count=struct.pack("<I", len(self.conns)),
                      chunk_count=struct.pack("<I", len(self.chunk_infos)))
        pad = 4096 - 4 - len(hdr) - 4
        self.out[self.header_pos:self.header_pos + 4096] = _record(hdr, b" " * pad)
        with open(self.path, "wb") as f:
            f.write(self.out)
        return bytes(self.out)


def write_event_bag(path, streams, infos=(), extras=True, msg_events=1000, msg_stamps=None, **kw):
    """streams: {topic: dict(x, y, t, p)} -- each cut into EventArrays of msg_events events (or at the indices msg_stamps[topic]
    gives, a list of (start, stop) slices, empty slices allowed) and interleaved by each message's last stamp with
    CameraInfo topics (infos: {topic: (width, height, model, D, K, R, P)}) and, with extras, Imu and Image topics.
    kw: BagWriter's."""
    msgs = []
    for topic, e in streams.items():
        n = len(e["t"])
        cuts = msg_stamps[topic] if msg_stamps and topic in msg_stamps else [(a, min(n, a + msg_events)) for a in range(0, n, msg_events)]
        for a, b in cuts:
            stamp = int(e["t"][b - 1]) if b > a else (int(e["t"][a - 1]) if a > 0 else 0)
            msgs.append((stamp, topic, "dvs_msgs/EventArray", event_array(e["x"][a:b], e["y"][a:b], e["t"][a:b], e["p"][a:b], stamp)))
    t_all = [m[0] for m in msgs] or [0]
    t_lo, t_hi = min(t_all), max(t_all)
    for topic, (W, H, model, D, K, R, P) in dict(infos).items():
        for k in range(3):
            msgs.append((t_lo + k * 10_000_000, topic, "sensor_msgs/CameraInfo", camera_info(W, H, model, D, K, R, P, t_lo)))
    if extras:
        for k, t in enumerate(np.linspace(t_lo, t_hi, 40).astype(np.int64)):
            msgs.append((int(t), "/dvs/imu", "sensor_msgs/Imu", imu(int(t), k)))
            if k % 4 == 0:
                msgs.append((int(t), "/dvs/image_raw", "sensor_msgs/Image", image(int(t), seq=k)))
    msgs.sort(key=lambda m: m[0])   # stable: each topic keeps its own order
    w = BagWriter(path, **kw)
    for t, topic, typ, payload in msgs:
        w.write(topic, typ, t, payload)
    return w.close()
