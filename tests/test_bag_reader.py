"""The ROS bag reader (include/esvo_b200/rosbag_events.hpp, through examples/bag_dump.cpp) against bags written by the
independent writer tests/rosbag_writer.py: every event, every takeBefore split, the CameraInfo rigs and the refusals.  CPU only."""
import os
import struct
import subprocess

import numpy as np
import pytest

import rosbag_writer as rw
from conftest import has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "esvo_b200", "_build")
L, R = "/davis/left/events", "/davis/right/events"
LI, RI = "/davis/left/camera_info", "/davis/right/camera_info"


def _compile(tmp_path_factory, name):
    exe = str(tmp_path_factory.mktemp("bin") / name)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", name + ".cpp"),
                           "-L" + BUILD, "-lesvo_b200", "-Wl,-rpath," + BUILD, "-o", exe])
    return exe


@pytest.fixture(scope="module")
def bag_dump(product_lib, tmp_path_factory):
    return _compile(tmp_path_factory, "bag_dump")


def _stream(n, seed, t0=1_600_000_000 * 10**9 + 999_000_000, ties=True):
    rng = np.random.default_rng(seed)
    dt = rng.integers(0, 3000, n) if ties else rng.integers(1, 3000, n)
    if ties:
        dt[rng.random(n) < 0.3] = 0                     # runs of equal stamps
    t = t0 + np.cumsum(dt).astype(np.int64)
    return dict(x=rng.integers(0, 346, n).astype(np.uint16), y=rng.integers(0, 260, n).astype(np.uint16), t=t,
                p=rng.integers(0, 2, n).astype(np.uint8))


def _dump_events(exe, bag, topic, tmp_path):
    out = tmp_path / "ev.bin"
    p = subprocess.run([exe, "events", str(bag), topic, str(out)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    raw = out.read_bytes()
    n = struct.unpack_from("<Q", raw)[0]
    rec = np.frombuffer(raw, rw.EVENT_DTYPE, n, 8)
    t = np.frombuffer(raw, np.int64, n, 8 + 13 * n)
    return rec, t


def _check_events(rec, t, e):
    assert rec.size == len(e["t"])
    assert np.array_equal(rec["x"], e["x"]) and np.array_equal(rec["y"], e["y"]) and np.array_equal(rec["polarity"], e["p"])
    assert np.array_equal(t, e["t"])
    assert np.array_equal(rec["sec"].astype(np.int64) * 10**9 + rec["nsec"], e["t"])


# chunk thresholds from one message per chunk to everything in one chunk; connection records in the chunks and in the index
# section only; message sizes 0, 1, 100 000 and mixed
@pytest.mark.parametrize("threshold,conn_in_chunks", [(1, True), (1, False), (4096, True), (200_000, False), (1 << 30, True)])
def test_every_event_decoded(bag_dump, tmp_path, threshold, conn_in_chunks):
    e = _stream(230_000, 1)
    r = _stream(30_000, 2)
    n = e["t"].size
    cuts = [(0, 0), (0, 1), (1, 1), (1, 100_001), (100_001, 100_001), (100_001, 100_002)]
    cuts += [(a, min(n, a + 7_777)) for a in range(100_002, n, 7_777)] + [(n, n)]
    bag = tmp_path / "b.bag"
    rw.write_event_bag(bag, {L: e, R: r}, msg_stamps={L: cuts}, msg_events=999, chunk_threshold=threshold, conn_in_chunks=conn_in_chunks)
    for topic, s in ((L, e), (R, r)):
        _check_events(*_dump_events(bag_dump, bag, topic, tmp_path), s)


def test_empty_and_single_event_topics(bag_dump, tmp_path):
    one = _stream(1, 3)
    none = dict(x=np.zeros(0, np.uint16), y=np.zeros(0, np.uint16), t=np.zeros(0, np.int64), p=np.zeros(0, np.uint8))
    bag = tmp_path / "b.bag"
    rw.write_event_bag(bag, {L: one, R: none}, msg_stamps={R: [(0, 0), (0, 0)]}, chunk_threshold=1)
    _check_events(*_dump_events(bag_dump, bag, L, tmp_path), one)
    _check_events(*_dump_events(bag_dump, bag, R, tmp_path), none)


def test_stamp_edges_decoded(bag_dump, tmp_path):
    """nsec = 999 999 999, sec near 2^32, polarity bytes 0, 1, 2, 255: stamps are sec * 1e9 + nsec in 64 bits."""
    sec = np.array([0, 1, 2**31, 2**32 - 2, 2**32 - 1, 2**32 - 1], np.uint32)
    nsec = np.array([999_999_999, 0, 999_999_999, 999_999_999, 0, 999_999_999], np.uint32)
    rec = np.zeros(sec.size, rw.EVENT_DTYPE)
    rec["sec"], rec["nsec"], rec["x"], rec["y"], rec["polarity"] = sec, nsec, [0, 65535, 346, 5, 6, 7], [260, 0, 65535, 1, 2, 3], [0, 1, 2, 255, 1, 0]
    bag = tmp_path / "b.bag"
    w = rw.BagWriter(bag, chunk_threshold=1)
    w.write(L, "dvs_msgs/EventArray", 10**9, rw.event_array_raw(rec[:3], 10**9))
    w.write(L, "dvs_msgs/EventArray", 2 * 10**9, rw.event_array_raw(rec[3:], 2 * 10**9))
    w.close()
    got, t = _dump_events(bag_dump, bag, L, tmp_path)
    assert got.tobytes() == rec.tobytes()
    assert t.tolist() == [int(s) * 10**9 + int(n) for s, n in zip(sec, nsec)]


def _take(exe, bag, topic, queries, tmp_path):
    qf, out = tmp_path / "q.bin", tmp_path / "take.bin"
    qf.write_bytes(np.asarray(queries, np.int64).tobytes())
    p = subprocess.run([exe, "take", str(bag), topic, str(qf), str(out)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    raw = out.read_bytes()
    k = np.frombuffer(raw, np.uint64, 2 * len(queries)).reshape(-1, 2)
    rec = np.frombuffer(raw, rw.EVENT_DTYPE, int(k[:, 1].sum()), 16 * len(queries))
    return k, rec


@pytest.mark.parametrize("msg_events", [1, 37, 1000])
def test_take_before_is_searchsorted(bag_dump, tmp_path, msg_events):
    """takeBefore(t) hands out exactly the events searchsorted(t, 'left') puts before t: ties at t stay for the next call,
    messages are split inside, empty messages are stepped over."""
    e = _stream(20_000, 4)
    n = e["t"].size
    cuts = [(a, min(n, a + msg_events)) for a in range(0, n, msg_events)]
    cuts = cuts[:3] + [(cuts[2][1], cuts[2][1])] * 2 + cuts[3:] + [(n, n)]     # empty messages in the middle and at the end
    bag = tmp_path / "b.bag"
    rw.write_event_bag(bag, {L: e}, msg_stamps={L: cuts}, chunk_threshold=3000)
    rng = np.random.default_rng(msg_events)
    t = e["t"]
    q = np.concatenate([t[rng.integers(0, n, 60)],                              # at an event's stamp: ties
                        t[rng.integers(0, n, 60)] + 1,                          # just after
                        rng.integers(t[0] - 10, t[-1] + 10, 60),
                        [t[0] - 1, t[0], t[msg_events - 1], t[msg_events], t[-1], t[-1] + 1, t[-1] + 1]])
    q = np.sort(q)
    k, rec = _take(bag_dump, bag, L, q, tmp_path)
    cum = np.searchsorted(t, q, "left")
    assert np.array_equal(np.cumsum(k[:, 1]), cum)
    assert rec["x"].tolist() == e["x"][: cum[-1]].tolist() and np.array_equal(rec["sec"].astype(np.int64) * 10**9 + rec["nsec"], t[: cum[-1]])
    assert (k[:, 0] <= k[:, 1]).all() and (k[k[:, 1] == 0, 0] == 0).all()   # no empty runs
    assert np.any(np.isin(q, t)) and np.any(k[:, 0] > 1)


def _calib_fields(c):
    from esvo_b200 import capi
    return bytes(memoryview(c).cast("B")) if isinstance(c, capi.Calib) else None


@pytest.mark.parametrize("rig", ["hkust", "dsec", "rpg", "upenn"])
def test_camera_info_gives_the_rig(bag_dump, product_lib, tmp_path, rig):
    """CameraInfo -> esvo_calib equals configs.rig_calibs field for field, and esvo_compute_rectify_tables gives identical
    tables from it (no GPU needed)."""
    from esvo_b200 import capi, configs
    rr = configs.RIGS[rig]
    infos = {}
    for topic, side in ((LI, "left"), (RI, "right")):
        c = rr[side]
        D = list(c["D"]) + ([0.0] if rr["model"] == "plumb_bob" and side == "right" else [])   # plumb_bob with k3 = 0
        infos[topic] = (rr["width"], rr["height"], rr["model"], D, c["K"], c["R"], c["P"])
    bag = tmp_path / "b.bag"
    rw.write_event_bag(bag, {L: _stream(100, 5)}, infos=infos, chunk_threshold=2000)
    for topic, want in zip((LI, RI), configs.rig_calibs(rig)):
        out = tmp_path / "calib.bin"
        p = subprocess.run([bag_dump, "calib", str(bag), topic, str(out)], capture_output=True, text=True)
        assert p.returncode == 0, p.stdout + p.stderr
        raw = out.read_bytes()
        got = capi.Calib.from_buffer_copy(raw[: capi.C.sizeof(capi.Calib)])
        assert bytes(got) == bytes(want)
        n = want.width * want.height
        off = capi.C.sizeof(capi.Calib)
        m1 = np.frombuffer(raw, np.float32, n, off); off += 4 * n
        m2 = np.frombuffer(raw, np.float32, n, off); off += 4 * n
        lut = np.frombuffer(raw, np.float64, 2 * n, off); off += 16 * n
        mask = np.frombuffer(raw, np.uint8, n, off)
        w1, w2, wl, wm = capi.compute_rectify_tables(product_lib, want)
        assert m1.tobytes() == w1.tobytes() and m2.tobytes() == w2.tobytes() and lut.tobytes() == wl.tobytes() and mask.tobytes() == wm.tobytes()


def _refusal(exe, bag, tmp_path, topic=L, mode="events"):
    p = subprocess.run([exe, mode, str(bag), topic, str(tmp_path / "x.bin")], capture_output=True, text=True)
    assert p.returncode == 3, (p.returncode, p.stdout + p.stderr)
    return p.stdout


def test_refusals(bag_dump, tmp_path):
    e = _stream(5000, 6)
    info = {LI: (346, 260, "plumb_bob", [0.1, 0.2, 0.0, 0.0], np.eye(3).ravel(), np.eye(3).ravel(), [1, 0, 1, 0, 0, 1, 1, 0, 0, 0, 1, 0])}
    for comp in ("bz2", "lz4"):
        bag = tmp_path / f"{comp}.bag"
        rw.write_event_bag(bag, {L: e}, chunk_threshold=4000, compression=comp)
        msg = _refusal(bag_dump, bag, tmp_path)
        assert "rosbag decompress" in msg and comp in msg, msg
    v12 = tmp_path / "v12.bag"
    v12.write_bytes(b"#ROSBAG V1.2\n" + b"\0" * 200)
    assert "V1.2" in _refusal(bag_dump, v12, tmp_path)
    bag = tmp_path / "ok.bag"
    raw = rw.write_event_bag(bag, {L: e}, infos=info, chunk_threshold=4000)
    cut = tmp_path / "cut.bag"
    rng = np.random.default_rng(0)
    for k in sorted(set(rng.integers(1, len(raw), 40).tolist()) | {5, 13, 4109, 4110, len(raw) - 1}):
        cut.write_bytes(raw[:k])
        msg = _refusal(bag_dump, cut, tmp_path)
        assert "truncated" in msg or "not a ROS bag" in msg, (k, msg)
    assert "not dvs_msgs/EventArray" in _refusal(bag_dump, bag, tmp_path, topic="/dvs/imu")
    assert "not dvs_msgs/EventArray" in _refusal(bag_dump, bag, tmp_path, topic=LI)
    assert "not sensor_msgs/CameraInfo" in _refusal(bag_dump, bag, tmp_path, topic=L, mode="calib")
    assert "no topic" in _refusal(bag_dump, bag, tmp_path, topic="/nothing")


def test_bag_system_builds_and_fails_cleanly_without_gpu(product_lib, tmp_path_factory, tmp_path):
    from esvo_b200 import configs
    exe = _compile(tmp_path_factory, "bag_system")
    if has_gpu():
        return
    rr = configs.RIGS["hkust"]
    infos = {t: (rr["width"], rr["height"], rr["model"], rr[s]["D"], rr[s]["K"], rr[s]["R"], rr[s]["P"]) for t, s in ((LI, "left"), (RI, "right"))}
    bag = tmp_path / "b.bag"
    rw.write_event_bag(bag, {L: _stream(500, 7), R: _stream(500, 8)}, infos=infos, chunk_threshold=2000)
    args = [exe, str(bag), L, R, LI, RI, str(tmp_path / "r.bin"), str(tmp_path / "traj.txt")]
    p = subprocess.run(args + ["--ticks", "3"], capture_output=True, text=True)
    assert p.returncode == 2 and "no CPU fallback" in p.stdout, p.stdout + p.stderr
    p = subprocess.run(args[:4] + ["/dvs/imu"] + args[5:], capture_output=True, text=True)   # a refused bag stops before the device
    assert p.returncode == 3 and "not sensor_msgs/CameraInfo" in p.stdout, p.stdout + p.stderr
