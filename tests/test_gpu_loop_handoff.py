"""Device-resident hand-off of the closed loop (include/esvo_b200.h: esvo_ts_history_*_dev, esvo_set_ts_pair_stored_dev,
esvo_map_publish_dev, esvo_track_adopt_map_dev, esvo_track_reset_dev) against the host forms on host copies of the same data:
the time-surface history against esvo_set_ts_pair with the images downloaded at each build, the published cloud against
frontend::packPointCloud over esvo_map_download, and the tracker on the adopted cloud against esvo_track_reset on a host copy."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from esvo_b200 import capi
from util import make_backends, scenario

pytestmark = pytest.mark.gpu

ERR_STATE = -5
CAP = 4                      # history capacity of the history tests


# ---------------------------------------------------------------- the new entry points
def _dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def reserve(g, cap):
    g._call("ts_history_reserve_dev", [C.c_size_t], cap)


def store(g, stamp):
    g._call("ts_history_store_dev", [C.c_int64], int(stamp))


def set_stored(g, stamp, T, ok=(0,)):
    T = np.ascontiguousarray(T, np.float64)
    return g._call("set_ts_pair_stored_dev", [C.c_int64, C.POINTER(C.c_double)], int(stamp), _dptr(T), ok=ok)


def publish(g, T, stamp):
    T = np.ascontiguousarray(T, np.float64); n = C.c_size_t(0)
    g._call("map_publish_dev", [C.POINTER(C.c_double), C.c_int64, C.POINTER(C.c_size_t)], _dptr(T), int(stamp), C.byref(n))
    return n.value


def published(g):
    """The published cloud, read back through a device buffer."""
    import torch
    buf = torch.zeros(3 * g.W * g.H, dtype=torch.float32, device="cuda")
    n = C.c_size_t(g.W * g.H); st = C.c_int64(0)
    g._call("map_published_cloud_dev", [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_int64)], C.c_void_p(buf.data_ptr()),
            C.byref(n), C.byref(st))
    return buf[: 3 * n.value].cpu().numpy().reshape(-1, 3), st.value


def adopt(g, stamp, ok=(0,)):
    n = C.c_size_t(0)
    rc = g._call("track_adopt_map_dev", [C.c_int64, C.POINTER(C.c_size_t)], int(stamp), C.byref(n), ok=ok)
    return rc, n.value


def reset_dev(g, Twr, Twc, ts_left=None):
    Tr = np.ascontiguousarray(Twr, np.float64); Tc = np.ascontiguousarray(Twc, np.float64)
    ts = None if ts_left is None else np.ascontiguousarray(ts_left, np.uint8)
    return g._call("track_reset_dev", [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_uint8)], _dptr(Tr), _dptr(Tc),
                   None if ts is None else ts.ctypes.data_as(C.POINTER(C.c_uint8)), ok=(0, 1))


def pack(p_cam, T):
    """frontend::packPointCloud: every row summed left to right from separately rounded products, then one f32 conversion."""
    p = np.asarray(p_cam, np.float64).reshape(-1, 3); T = np.asarray(T, np.float64).reshape(4, 4)
    return np.stack([T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1] + T[r, 2] * p[:, 2] + T[r, 3] for r in range(3)], axis=1).astype(np.float32)


def _fl(x):
    return float(x)          # Fraction -> nearest double


def pack_fma(p, T):
    """The same row as an FMA-contracting compiler emits it: fma(T2, p2, fma(T1, p1, T0 p0)) + T3 (exact products)."""
    out = np.empty((p.shape[0], 3), np.float32)
    T = np.asarray(T, np.float64).reshape(4, 4)
    for i, q in enumerate(np.asarray(p, np.float64).reshape(-1, 3)):
        for r in range(3):
            a = _fl(Fraction(T[r, 1]) * Fraction(q[1]) + Fraction(T[r, 0] * q[0]))
            a = _fl(Fraction(T[r, 2]) * Fraction(q[2]) + Fraction(a))
            out[i, r] = np.float32(a + T[r, 3])
    return out


def fma_sensitive_pose(p_cam, T):
    """T with its translation chosen so that, for one element per row, the sum without FMA and the FMA-contracted sum round to
    different floats: the translation puts that element's world coordinate next to a float32 rounding midpoint.  Returns the
    pose and the indices of the elements."""
    T = np.array(T, np.float64).reshape(4, 4)
    p = np.asarray(p_cam, np.float64).reshape(-1, 3)
    picks = []
    for r in range(3):
        found = False
        for i in range(p.shape[0]):
            a = T[r, 0] * p[i, 0] + T[r, 1] * p[i, 1] + T[r, 2] * p[i, 2]
            b = _fl(Fraction(T[r, 1]) * Fraction(p[i, 1]) + Fraction(T[r, 0] * p[i, 0]))
            b = _fl(Fraction(T[r, 2]) * Fraction(p[i, 2]) + Fraction(b))
            if a == b:
                continue
            if abs(a) < 1e-3:
                continue
            # a float32 rounding midpoint near a / 4: with t in [-a, -a / 2] the sums a + t and b + t are exact (Sterbenz),
            # so they keep their difference and can sit on either side of the midpoint
            f = np.float32(a / 4)
            mid = (float(f) + float(np.nextafter(f, np.float32(np.inf)))) / 2   # exactly representable in f64
            t0 = mid - (a + b) / 2
            for k in range(-64, 65):
                t = float(np.nextafter(t0, np.inf if k > 0 else -np.inf)) if k else t0
                for _ in range(abs(k) - 1):
                    t = float(np.nextafter(t, np.inf if k > 0 else -np.inf))
                if np.float32(a + t) != np.float32(b + t):
                    T[r, 3] = t; picks.append(i); found = True
                    break
            if found:
                break
        assert found, f"no element of the map lets row {r} tell FMA from no FMA"
    return T, picks


# ---------------------------------------------------------------- 1. history
@pytest.mark.parametrize("rig", ["hkust", "dsec"])
@pytest.mark.parametrize("smooth", [0, 1])
@pytest.mark.parametrize("k", [CAP - 1, CAP, CAP + 1])
def test_history_hands_over_the_requested_pair(oracle_lib, product_lib, rig, smooth, k):
    """K builds into a history of CAP pairs: every stored stamp gives the BM seeds and evaluation count of esvo_set_ts_pair with
    the images downloaded at that build; dropped and unknown stamps are refused and the context stays usable."""
    s = scenario(rig, n_seeds=800)

    def tweak(p):
        p.smooth_time_surface = smooth
    _, g = make_backends(rig, oracle_lib, product_lib, tweak)
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
    reserve(g, CAP)
    stamps = [s["t_ts_ns"] - (k - 1 - j) * 2_000_000 for j in range(k)]
    imgs = {}
    for t in stamps:
        imgs[t] = (g.ts_build(0, t, want_idx=False)[1].copy(), g.ts_build(1, t, want_idx=False)[1].copy())
        store(g, t)
    # the pairs differ from stamp to stamp, so handing over the wrong one shows
    assert all(not np.array_equal(imgs[a][0], imgs[b][0]) for a, b in zip(stamps, stamps[1:]))
    T = s["T_world_left"]
    sd = s["seeds"]
    kept = stamps[-CAP:]
    for t in stamps[: len(stamps) - len(kept)] + [stamps[-1] + 1, stamps[0] - 1]:
        assert set_stored(g, t, T, ok=(0, ERR_STATE)) == ERR_STATE, t
    for t in reversed(kept):
        set_stored(g, t, T)
        seeds_d, ev_d = g.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        g.set_ts_pair(imgs[t][0], imgs[t][1], T)
        seeds_h, ev_h = g.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        assert seeds_h.size > 0
        assert ev_d == ev_h and seeds_d.tobytes() == seeds_h.tobytes(), f"stamp {t}: {seeds_d.size} / {seeds_h.size} seeds"
    # the stored pair also feeds the SGM start-up (esvo_sgbm_compute(NULL, NULL))
    set_stored(g, kept[0], T)
    assert np.array_equal(g.sgbm_compute(), g.sgbm_compute(imgs[kept[0]][0], imgs[kept[0]][1]))


def test_history_store_refused_without_reservation(oracle_lib, product_lib):
    s = scenario("hkust", n_seeds=200)
    _, g = make_backends("hkust", oracle_lib, product_lib)
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
    g.ts_build(0, s["t_ts_ns"]); g.ts_build(1, s["t_ts_ns"])
    with pytest.raises(capi.EsvoError) as ei:
        store(g, s["t_ts_ns"])
    assert ei.value.code == ERR_STATE
    reserve(g, 2); store(g, s["t_ts_ns"]); reserve(g, 0)
    assert set_stored(g, s["t_ts_ns"], s["T_world_left"], ok=(0, ERR_STATE)) == ERR_STATE


# ---------------------------------------------------------------- 2. publish
def _mapped(rig, oracle_lib, product_lib, frames, tweak=None, n_seeds=1500):
    s = scenario(rig, n_seeds=n_seeds)
    _, g = make_backends(rig, oracle_lib, product_lib, tweak)
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
    g.ts_build(0, s["t_ts_ns"]); g.ts_build(1, s["t_ts_ns"])
    sd = s["seeds"]
    for f in range(frames):
        g.set_ts_pair(None, None, s["T_world_left"])
        g.mapping_at_time(sd["x"][f::frames] if frames > 1 else sd["x"], sd["y"][f::frames] if frames > 1 else sd["y"],
                          sd["t"][f::frames] if frames > 1 else sd["t"], s["pose_t"], s["poses"])
    return s, g


def _check_publish(g, T, stamp, fma_probe=True):
    m = g.map_download()
    if fma_probe and m.size:
        T, picks = fma_sensitive_pose(m["p_cam"], T)
    n = publish(g, T, stamp)
    cloud, st = published(g)
    want = pack(m["p_cam"], T)
    assert n == m.size == cloud.shape[0] and st == stamp
    assert cloud.tobytes() == want.tobytes(), f"{(cloud != want).any(axis=1).sum()} of {n} points differ"
    if fma_probe and m.size:
        fused = pack_fma(m["p_cam"][picks], T)
        for r, i in enumerate(picks):        # present in the cloud, and an FMA would have rounded them differently
            assert cloud[i, r] == want[i, r] and fused[r, r] != want[i, r], (r, i)
    return n


def test_publish_after_sgm_startup(oracle_lib, product_lib):
    s = scenario("hkust", n_seeds=1500)
    _, g = make_backends("hkust", oracle_lib, product_lib)
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
    g.ts_build(0, s["t_ts_ns"]); g.ts_build(1, s["t_ts_ns"])
    g.set_ts_pair(None, None, np.eye(4).ravel())
    disp = g.sgbm_compute()
    ev = s["left"]
    n_pts, accepted = g.init_from_disparity(disp, ev["x"][-1001:], ev["y"][-1001:], np.eye(4).ravel(), 1)
    assert accepted and n_pts > 100
    assert _check_publish(g, s["T_world_left"], 7) > 100


@pytest.mark.parametrize("rig", ["hkust", "dsec"])
def test_publish_after_working_frames_with_regularisation(oracle_lib, product_lib, rig):
    def tweak(p):
        p.regularization = 1
    s, g = _mapped(rig, oracle_lib, product_lib, 3, tweak)
    assert _check_publish(g, s["T_world_left"], s["t_ts_ns"]) > 100
    # the map of separate fusions (more than one fold: the element list is ranked by creation key instead)
    m = g.map_download()
    T = m[0]["T_world_cam"]
    g.fuse(m[: m.size // 2], T, 0, True)
    g.fuse(m[m.size // 2:], T, 0, False)
    assert _check_publish(g, s["T_world_left"], 11) > 100
    # elements removed after the fold (SmartGrid::clean on its own): the creator bits no longer describe the map
    g.fuse(m, T, 0, True)
    g.map_clean(1e9, -1.0, float(np.median(m["inv_depth"])), 0.0)    # drops the nearer half
    assert 0 < _check_publish(g, s["T_world_left"], 13) < m.size
    # a second publish replaces the first
    assert _check_publish(g, np.eye(4).ravel(), 12, fma_probe=False) > 100


def test_publish_empty_map(oracle_lib, product_lib):
    _, g = make_backends("hkust", oracle_lib, product_lib)
    with pytest.raises(capi.EsvoError) as ei:
        published(g)
    assert ei.value.code == ERR_STATE
    g.fuse(np.zeros(0, capi.DEPTH_POINT_DTYPE), np.eye(4).ravel(), 0, True)
    assert publish(g, np.eye(4).ravel(), 3) == 0
    cloud, st = published(g)
    assert cloud.shape == (0, 3) and st == 3
    assert adopt(g, 3)[1] == 0
    assert reset_dev(g, np.eye(4).ravel(), np.eye(4).ravel()) == 1


# ---------------------------------------------------------------- 3. tracker
def _tracker_ctx(oracle_lib, product_lib, max_reg, subset=None, batch=None):
    """A context with a mapped hkust scene whose map (or the map of its first `subset` elements, fused alone) is published at
    stamp 5."""
    def tweak(p):
        p.trk_max_registration_points = max_reg
        if batch is not None:
            p.trk_batch_size = batch
    s, g = _mapped("hkust", oracle_lib, product_lib, 1, tweak, n_seeds=4000)
    if subset is not None:
        m = g.map_download()
        g.fuse(m[:subset], m[0]["T_world_cam"], 0, True)
    n = publish(g, s["T_world_left"], 5)
    return s, g, n


def _run(g, forms, clouds, Twr, Twc0, seed=3):
    """Consecutive reset + solve passes; forms[i] 'h' resets from clouds['h'] (host, permuted in place), 'd' from the adopted
    cloud ('x' from clouds['x'], the host stand-in for the adopted one)."""
    g.track_srand(seed)
    out, Twc = [], np.asarray(Twc0, np.float64).ravel()
    for f in forms:
        rc = reset_dev(g, Twr, Twc) if f == "d" else g.track_reset(clouds[f], Twr, Twc, None)
        if rc == 1:
            out.append(("not enough points",))
            continue
        T, st = g.track_solve(True)
        out.append((T.tobytes(), st["nfev"], st["n_iter"], st["n_points"]))
        Twc = T.ravel()
    return out


@pytest.mark.parametrize("case", ["below", "at", "above", "batch-1"])
def test_tracker_on_the_adopted_cloud(oracle_lib, product_lib, case):
    batch = 500                                       # hkust BATCH_SIZE
    if case == "batch-1":                             # a smaller map (the same on every context), BATCH_SIZE one above its size
        _, _, n1 = _tracker_ctx(oracle_lib, product_lib, 2000, subset=150)
        batch = n1 + 1
        assert batch <= 1024
        s, g, n = _tracker_ctx(oracle_lib, product_lib, 2000, subset=150, batch=batch)
        assert n == batch - 1
    else:
        s, g, n0 = _tracker_ctx(oracle_lib, product_lib, 2000)
        max_reg = {"below": n0 + 37, "at": n0, "above": (n0 + batch) // 2}[case]
        s, g, n = _tracker_ctx(oracle_lib, product_lib, max_reg)
        assert n == n0 and n > batch + 40, n
    cloud, _ = published(g)
    assert adopt(g, 5)[1] == n
    Twr = s["T_world_left"]
    Twc = np.asarray(Twr, np.float64).reshape(4, 4).copy(); Twc[0, 3] += 0.01
    dev = _run(g, "ddddd", {}, Twr, Twc)
    host = _run(g, "hhhhh", {"h": cloud.copy()}, Twr, Twc)
    assert dev == host, case
    if case == "batch-1":
        assert dev == [("not enough points",)] * 5
    else:
        assert all(len(r) == 4 for r in dev)
    # one rand() stream across forms: host and device resets alternating on two clouds equal the same on two host clouds
    adopt(g, 5)
    mixed = _run(g, "hdhdhd", {"h": cloud.copy()}, Twr, Twc)
    allhost = _run(g, "hxhxhx", {"h": cloud.copy(), "x": cloud.copy()}, Twr, Twc)
    assert mixed == allhost


def test_adoption_is_a_snapshot(oracle_lib, product_lib):
    """A publish after the adoption does not change the tracker's cloud; adopting needs the newest stamp."""
    s, g, n = _tracker_ctx(oracle_lib, product_lib, 2000)
    cloud, _ = published(g)
    adopt(g, 5)
    assert adopt(g, 4, ok=(0, ERR_STATE))[0] == ERR_STATE
    adopt(g, 5)
    T = np.asarray(s["T_world_left"], np.float64).reshape(4, 4).copy(); T[:3, 3] += 0.5
    publish(g, T, 6)                                  # another cloud, same map: every point moved
    Twr = s["T_world_left"]
    Twc = np.asarray(Twr, np.float64).reshape(4, 4).copy(); Twc[1, 3] -= 0.01
    assert _run(g, "ddd", {}, Twr, Twc) == _run(g, "hhh", {"h": cloud.copy()}, Twr, Twc)
