"""Packed-event ingest on the H100 (esvo_ts_push_event_array / _dev, ts_ingest_packed_kernel) against the SoA push
(esvo_ts_push_events) on the same events: after every push sequence the index grid and the published image of esvo_ts_build
are byte-identical, build refusals (order flag, folded log) are the same, and the event windows read from the log agree.
The closed loop from a bag (examples/bag_system.cpp) against examples/system_loop.cpp on the same scenario."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rosbag_writer as rw

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "esvo_b200", "_build")
ERR_CAPACITY, ERR_UNSUPPORTED = -4, -6
T0 = 1_600_000_000 * 10**9 + 123_456_789


def _ctx(lib, ignore_polarity=0):
    from esvo_b200 import capi, configs
    l, r = configs.rig_calibs("hkust")
    p = configs.params_for("hkust", lib)
    p.ignore_polarity = ignore_polarity
    return capi.Backend(lib, l, r, p)


def _build(b, cam, T):
    idx = np.empty(b.W * b.H, np.int64); img = np.empty(b.W * b.H, np.uint8)
    rc = b._call("ts_build", [C.c_int, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_uint8)], cam, int(T),
                 idx.ctypes.data_as(C.POINTER(C.c_int64)), img.ctypes.data_as(C.POINTER(C.c_uint8)), ok=(0, ERR_UNSUPPORTED))
    return rc, idx, img


def _stream(n, seed, t0=T0, x_max=346, y_max=260):
    rng = np.random.default_rng(seed)
    dt = rng.integers(0, 2000, n)
    dt[rng.random(n) < 0.3] = 0
    return dict(x=rng.integers(0, x_max, n).astype(np.uint16), y=rng.integers(0, y_max, n).astype(np.uint16),
                t=(t0 + np.cumsum(dt)).astype(np.int64), p=rng.integers(0, 2, n).astype(np.uint8))


def _cut(e, a, b):
    return {k: v[a:b] for k, v in e.items()}


def _records(e):
    r = np.empty(len(e["t"]), rw.EVENT_DTYPE)
    t = np.asarray(e["t"], np.int64)
    r["x"], r["y"], r["sec"], r["nsec"], r["polarity"] = e["x"], e["y"], t // 10**9, t % 10**9, e["p"]
    return r


class Pair:
    """The SoA context and the packed context, fed the same events."""

    def __init__(self, lib, form="host", ignore_polarity=0, offset=0, seed=0):
        self.soa, self.pk = _ctx(lib, ignore_polarity), _ctx(lib, ignore_polarity)
        self.form, self.offset, self.rng = form, offset, np.random.default_rng(seed)

    def push(self, cam, e=None, records=None, ok=(0,)):
        rec = _records(e) if records is None else records
        p01 = (rec["polarity"] != 0).astype(np.uint8)
        t = rec["sec"].astype(np.int64) * 10**9 + rec["nsec"].astype(np.int64)
        from esvo_b200 import capi
        try:
            self.soa.ts_push_events(cam, rec["x"], rec["y"], t, p01)
            rc_s = 0
        except capi.EsvoError as err:
            if err.code not in ok:
                raise
            rc_s = err.code
        raw = rec.tobytes()
        if self.form == "host":   # several runs at odd host addresses
            buf = bytearray(len(raw) + 16)
            buf[self.offset:self.offset + len(raw)] = raw
            mv = memoryview(buf)[self.offset:self.offset + len(raw)]
            k = sorted(set(self.rng.integers(0, rec.size + 1, 3).tolist()) | {0, rec.size})
            runs = [mv[13 * a:13 * b] for a, b in zip(k[:-1], k[1:])] + [b""]
            runs = [np.frombuffer(r, np.uint8) for r in runs]
            rc_p = self.pk.ts_push_event_array(cam, runs, ok=ok)
        else:                     # device memory at a byte offset
            import torch
            d = torch.zeros(len(raw) + 16, dtype=torch.uint8, device="cuda")
            d[self.offset:self.offset + len(raw)] = torch.from_numpy(np.frombuffer(raw, np.uint8).copy()).cuda()
            torch.cuda.synchronize()
            rc_p = self.pk.ts_push_event_array_dev(cam, d.data_ptr() + self.offset, rec.size, ok=ok)
            self.pk._call("sync", [])
            del d
        assert rc_s == rc_p, (rc_s, rc_p)
        return rc_s

    def same(self, cam, T):
        rs, i_s, m_s = _build(self.soa, cam, T)
        rp, i_p, m_p = _build(self.pk, cam, T)
        assert rs == rp, (rs, rp, T)
        if rs == 0:
            assert i_s.tobytes() == i_p.tobytes() and m_s.tobytes() == m_p.tobytes(), T
        return rs


@pytest.mark.parametrize("form", ["host", "dev"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 4095, 4096, 65537])
def test_packed_equals_soa_sizes(product_lib, n, form):
    e = _stream(n, n)
    pr = Pair(product_lib, form, offset=n % 16)
    for cam in (0, 1):
        pr.push(cam, e)
        assert pr.same(cam, e["t"][-1] + 1) == 0
        assert pr.same(cam, e["t"][n // 2]) == 0          # T inside the stream: the general path reads the log
    e2 = _stream(n, n + 1, t0=int(e["t"][-1]))           # a second push on top
    pr.push(0, e2)
    assert pr.same(0, e2["t"][-1] + 1) == 0 and pr.same(0, e["t"][-1]) == 0


@pytest.mark.parametrize("form", ["host", "dev"])
@pytest.mark.parametrize("offset", range(16))
def test_packed_equals_soa_offsets(product_lib, offset, form):
    e = _stream(4097 + offset, 100 + offset)
    pr = Pair(product_lib, form, offset=offset, seed=offset)
    pr.push(0, e)
    assert pr.same(0, e["t"][-1] + 1) == 0


def test_polarity_bytes_and_coordinates(product_lib):
    """Polarity bytes 0, 1, 2, 255 (a ROS bool is byte != 0) with polarity in the image; x = W, y = H and 65 535 are logged
    and counted but not scattered."""
    for form in ("host", "dev"):
        e = _stream(5000, 7)
        rng = np.random.default_rng(8)
        e["p"] = rng.choice(np.array([0, 1, 2, 255], np.uint8), e["p"].size)
        k = rng.choice(e["t"].size, 400, replace=False)
        e["x"][k[:100]] = 346; e["y"][k[100:200]] = 260; e["x"][k[200:300]] = 65535; e["y"][k[300:]] = 65535
        pr = Pair(product_lib, form, ignore_polarity=0, offset=3)
        pr.push(0, e)
        assert pr.same(0, e["t"][-1] + 1) == 0 and pr.same(0, e["t"][2500]) == 0
        rc, idx, img = _build(pr.pk, 0, e["t"][-1] + 1)
        assert len(np.unique(img)) > 2                   # both polarities reach the image


def test_stamp_edges(product_lib):
    """nsec = 999 999 999 and sec up to 2^32 - 1: stamps are sec * 1e9 + nsec in 64 bits (ros::Time::toNSec)."""
    n = 3000
    rng = np.random.default_rng(9)
    rec = np.zeros(n, rw.EVENT_DTYPE)
    sec = np.sort(rng.integers(2**32 - 40, 2**32, n)).astype(np.uint32)
    rec["sec"] = sec
    rec["nsec"] = np.where(rng.random(n) < 0.5, 999_999_999, 0)
    rec["nsec"][1:][sec[1:] == sec[:-1]] = np.maximum.accumulate(rec["nsec"])[1:][sec[1:] == sec[:-1]]
    t = rec["sec"].astype(np.int64) * 10**9 + rec["nsec"]
    assert (np.diff(t) >= 0).all()
    rec["x"] = rng.integers(0, 346, n); rec["y"] = rng.integers(0, 260, n); rec["polarity"] = rng.integers(0, 2, n)
    pr = Pair(product_lib, "host")
    pr.push(0, records=rec)
    assert pr.same(0, t[-1] + 1) == 0
    assert pr.same(0, t[-1] - 500_000_000) == 0          # the split falls on nsec = 999 999 999 / 0 boundaries
    rc, idx, _ = _build(pr.pk, 0, t[-1] + 1)
    assert (idx >= 0).sum() > 1000


@pytest.mark.parametrize("case", ["inside-17", "warp-32", "block-256", "across", "across-tie", "ordered"])
def test_order_flag_like_soa(product_lib, case):
    """The order flag goes up exactly when the SoA push raises it: inside a push (inside a warp, at a warp's first record, at
    a block's first record) and at the first record of a push against the newest stamp before it."""
    e = _stream(3000, 11)
    e["t"] = (T0 + np.arange(3000) * 1000).astype(np.int64)
    first, second = _cut(e, 0, 1500), _cut(e, 1500, 3000)
    if case.startswith(("inside", "warp", "block")):
        i = int(case.split("-")[1])
        second["t"] = second["t"].copy(); second["t"][i] = second["t"][i - 1] - 1
    elif case == "across":
        second["t"] = second["t"] - 1000 * 2                    # first record older than the newest of the first push
    elif case == "across-tie":
        second["t"] = second["t"] - 1000                        # first record ties with the newest: ordered
    for form in ("host", "dev"):
        pr = Pair(product_lib, form)
        pr.push(0, first)
        pr.push(0, second)
        rc = pr.same(0, int(second["t"].max()) + 1)
        assert rc == (0 if case in ("ordered", "across-tie") else ERR_UNSUPPORTED), (case, form, rc)


def test_unordered_mode(product_lib):
    e = _stream(20_000, 12)
    rng = np.random.default_rng(13)
    e["t"] = e["t"] + rng.integers(-30_000, 30_000, e["t"].size)   # jittered: out of order everywhere
    e["t"][e["t"] < 0] = 0
    for form in ("host", "dev"):
        pr = Pair(product_lib, form)
        for b in (pr.soa, pr.pk):
            b.ts_set_unordered_input(0, 1)
        for a, z in ((0, 1), (1, 4096), (4096, 20_000)):
            pr.push(0, _cut(e, a, z))
            assert pr.same(0, int(e["t"][:z].max()) + 1) == 0
        assert pr.same(0, int(np.median(e["t"]))) == 0


def test_fold_over_a_long_sequence(product_lib):
    """7.5 M events in pushes of up to 1.5 M fold the resident log; builds at the newest stamp and refused builds before the
    folded part agree after every push."""
    n = 7_500_000
    rng = np.random.default_rng(14)
    e = dict(x=rng.integers(0, 346, n).astype(np.uint16), y=rng.integers(0, 260, n).astype(np.uint16),
             t=(T0 + np.cumsum(rng.integers(0, 3, n))).astype(np.int64), p=rng.integers(0, 2, n).astype(np.uint8))
    pr = Pair(product_lib, "host")
    cuts = [0, 1_500_000, 1_500_001, 3_000_000, 4_500_000, 6_000_000, n]
    refused = 0
    for a, z in zip(cuts[:-1], cuts[1:]):
        pr.push(0, _cut(e, a, z))
        assert pr.same(0, e["t"][z - 1] + 1) == 0
        refused += pr.same(0, e["t"][max(0, z - 3_000_000)]) == ERR_UNSUPPORTED
    assert refused >= 1


def test_half_log_refusal(product_lib):
    """A batch larger than half the resident log (2 Mi events) is refused by both forms and changes nothing."""
    e = _stream(2 * 2**20 + 1, 15)
    for form in ("host", "dev"):
        pr = Pair(product_lib, form)
        small = _stream(1000, 16, t0=int(e["t"][0]) - 10**7)
        pr.push(0, small)
        assert pr.push(0, e, ok=(ERR_CAPACITY,)) == ERR_CAPACITY
        assert pr.same(0, small["t"][-1] + 1) == 0
        pr.push(0, _cut(e, 0, 2**21))                       # exactly half the log is taken
        assert pr.same(0, e["t"][2**21 - 1] + 1) == 0


def test_event_windows_after_packed_pushes(product_lib):
    """esvo_events_window_dev / esvo_events_lower_bound_dev read the log the packed pushes wrote: same answers as after the
    SoA pushes."""
    e = _stream(60_000, 17)
    pr = Pair(product_lib, "host")
    for a, z in ((0, 10_000), (10_000, 10_000), (10_000, 35_000), (35_000, 60_000)):
        if z > a:
            pr.push(0, _cut(e, a, z))
    for b in (pr.soa, pr.pk):
        _build(b, 0, e["t"][-1] + 1)
    t = e["t"]
    for front, tb, te, budget, denoise in ((0, t[100], t[-1], 1000, 0), (0, t[20_000], t[-1], 1001, 1), (5000, t[0], t[30_000], 60_000, 0)):
        rs = pr.soa.events_window_dev(0, front, tb, te, budget, denoise, 100_000)
        rp = pr.pk.events_window_dev(0, front, tb, te, budget, denoise, 100_000)
        assert rs == rp
        xs, ys, ts = pr.soa.events_selected_dev(); xp, yp, tp = pr.pk.events_selected_dev()
        assert np.array_equal(xs, xp) and np.array_equal(ys, yp) and np.array_equal(ts, tp)
    q = np.sort(np.concatenate([t[::997], t[::1999] + 1]))
    for k in range(0, q.size, 64):                        # at most 64 stamps per call
        rs, i_s = pr.soa.events_lower_bound_dev(0, 0, q[k:k + 64])
        rp, i_p = pr.pk.events_lower_bound_dev(0, 0, q[k:k + 64])
        assert rs == rp == 0 and np.array_equal(i_s, i_p)


# ---------------------------------------------------------------- the closed loop from a bag
def _compile(tmp_path, name):
    exe = str(tmp_path / name)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", name + ".cpp"),
                           "-L" + BUILD, "-lesvo_b200", "-Wl,-rpath," + BUILD, "-o", exe])
    return exe


@pytest.mark.parametrize("scene", ["dense", "mapping"])
def test_bag_system_equals_system_loop(product_lib, tmp_path, scene):
    """The scenes of tests/test_system_loop.py (seed 2, hkust) written into bags with small chunks and extra topics:
    bag_system.cpp gives the tick records, trajectory file and final map of system_loop.cpp, byte for byte."""
    import indep_system as isy
    from esvo_b200 import configs
    import test_system_loop as tsl
    s = tsl._stream(scene)
    t0, n = tsl._ticks(s)
    scen, res_a, traj_a = tmp_path / "scen.bin", tmp_path / "a.bin", tmp_path / "a.txt"
    isy.write_scenario(scen, 346, 260, t0, tsl.DT_NS, n, s["left"], s["right"])
    p = subprocess.run([_compile(tmp_path, "system_loop"), str(scen), str(res_a), str(traj_a)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    rr = configs.RIGS["hkust"]
    L, R, LI, RI = "/davis/left/events", "/davis/right/events", "/davis/left/camera_info", "/davis/right/camera_info"
    infos = {t: (rr["width"], rr["height"], rr["model"], rr[sd]["D"], rr[sd]["K"], rr[sd]["R"], rr[sd]["P"]) for t, sd in ((LI, "left"), (RI, "right"))}
    bag = tmp_path / "scene.bag"
    rw.write_event_bag(bag, {L: s["left"], R: s["right"]}, infos=infos, msg_events=1500, chunk_threshold=64 * 1024)
    res_b, traj_b = tmp_path / "b.bin", tmp_path / "b.txt"
    p = subprocess.run([_compile(tmp_path, "bag_system"), str(bag), L, R, LI, RI, str(res_b), str(traj_b), "--t0-ns", str(t0),
                        "--dt-ns", str(tsl.DT_NS), "--ticks", str(n)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    print(p.stdout.strip())
    a, b = isy.parse_result(res_a), isy.parse_result(res_b)
    keys = ["t", "status", "has_pose", "T"]
    assert a[0].size == b[0].size == n and a[3] == b[3] == 0
    for k in keys:
        assert a[0][k].tobytes() == b[0][k].tobytes(), k
    assert a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes()
    assert traj_a.read_bytes() == traj_b.read_bytes() and len(traj_a.read_bytes()) > 0
