"""Hot pixels at the packed ingest on the H100 (include/esvo_b200_hotpix.h, hotpix.cu): the counts equal np.bincount over the
in-image records, the mask equals the rule restated in numpy bit for bit, a masked push equals an unmasked push of the records
numpy prefiltered with that mask, and bag_system --hot-pixels equals system_loop on the prefiltered streams."""
import math
import os
import subprocess

import numpy as np
import pytest

import rosbag_writer as rw
from test_gpu_bag_ingest import T0, _build, _compile, _records, _stream

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_UNSUPPORTED = -1, -4, -6
HALF_LOG = 2 * 2**20


def _ctx(lib, rig="hkust", ignore_polarity=0):
    from esvo_b200 import capi, configs
    l, r = configs.rig_calibs(rig)
    p = configs.params_for(rig, lib)
    p.ignore_polarity = ignore_polarity
    return capi.Backend(lib, l, r, p)


def _bincount(rec, W, H):
    x, y = rec["x"].astype(np.int64), rec["y"].astype(np.int64)
    ok = (x < W) & (y < H)
    return np.bincount(y[ok] * W + x[ok], minlength=W * H).astype(np.uint64)


def _rule(c, k):
    """The selection rule of include/esvo_b200_hotpix.h: exact integer sums, each rounded once to double, then IEEE double."""
    c = np.asarray(c).ravel()
    n = float(c.size)
    s1 = int(c.astype(object).sum())
    s2 = int((c.astype(object) ** 2).sum())
    mu = float(s1) / n
    sigma = math.sqrt(max(0.0, float(s2) / n - mu * mu))
    return (c.astype(np.float64) > mu + k * sigma).astype(np.uint8)


def _host_runs(raw, offset, rng):
    """raw bytes as several runs at an odd host address (offset 0-15), one of them empty."""
    buf = bytearray(len(raw) + 16)
    buf[offset:offset + len(raw)] = raw
    mv = memoryview(buf)[offset:offset + len(raw)]
    n = len(raw) // 13
    k = sorted(set(rng.integers(0, n + 1, 3).tolist()) | {0, n})
    return [np.frombuffer(mv[13 * a:13 * b], np.uint8) for a, b in zip(k[:-1], k[1:])] + [np.zeros(0, np.uint8)]


def _dev(raw, offset):
    import torch
    d = torch.zeros(len(raw) + 16, dtype=torch.uint8, device="cuda")
    if raw:
        d[offset:offset + len(raw)] = torch.from_numpy(np.frombuffer(raw, np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    return d


def _count(b, cam, rec, form="host", offset=0, seed=0):
    raw = rec.tobytes()
    if form == "host":
        b.hotpix_count_event_array(cam, _host_runs(raw, offset, np.random.default_rng(seed)))
    else:
        d = _dev(raw, offset)
        b.hotpix_count_event_array_dev(cam, d.data_ptr() + offset, rec.size)
        b._call("sync", [])
        del d


def _push(b, cam, rec, form="host", offset=0, seed=0, ok=(0,)):
    raw = rec.tobytes()
    if form == "host":
        return b.ts_push_event_array(cam, _host_runs(raw, offset, np.random.default_rng(seed)), ok=ok)
    d = _dev(raw, offset)
    rc = b.ts_push_event_array_dev(cam, d.data_ptr() + offset, rec.size, ok=ok)
    b._call("sync", [])
    del d
    return rc


def _with_outside(rec, W, H, seed):
    """Some records outside the image: x = W, y = H, 65 535 -- neither counted nor dropped."""
    rec = rec.copy()
    rng = np.random.default_rng(seed)
    if rec.size >= 8:
        k = rng.choice(rec.size, max(4, rec.size // 50), replace=False)
        q = np.array_split(k, 4)
        rec["x"][q[0]] = W; rec["y"][q[1]] = H; rec["x"][q[2]] = 65535; rec["y"][q[3]] = 65535
    return rec


# ---------------------------------------------------------------- counts
@pytest.mark.parametrize("rig", ["hkust", "dsec"])
@pytest.mark.parametrize("form", ["host", "dev"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 4095, 65537])
def test_counts_equal_bincount_sizes(product_lib, n, form, rig):
    b = _ctx(product_lib, rig)
    rec = _with_outside(_records(_stream(n, n, x_max=b.W, y_max=b.H)), b.W, b.H, n)
    for cam in (0, 1):
        _count(b, cam, rec, form, offset=n % 16, seed=cam)
        c, m = b.hotpix_read(cam)
        assert np.array_equal(c.ravel(), _bincount(rec, b.W, b.H)) and not m.any()
    # accumulation over several calls
    rec2 = _records(_stream(3 * n + 5, n + 1, x_max=b.W, y_max=b.H))
    for a, z in ((0, n), (n, 3 * n), (3 * n, 3 * n + 5)):
        _count(b, 0, rec2[a:z], form, offset=(a + 7) % 16)
    c, _ = b.hotpix_read(0)
    assert np.array_equal(c.ravel(), _bincount(rec, b.W, b.H) + _bincount(rec2, b.W, b.H))


@pytest.mark.parametrize("form", ["host", "dev"])
@pytest.mark.parametrize("offset", range(16))
def test_counts_equal_bincount_offsets(product_lib, offset, form):
    b = _ctx(product_lib)
    rec = _with_outside(_records(_stream(4097 + offset, 200 + offset)), b.W, b.H, offset)
    _count(b, 1, rec, form, offset=offset, seed=offset)
    c, _ = b.hotpix_read(1)
    assert np.array_equal(c.ravel(), _bincount(rec, b.W, b.H))


@pytest.mark.parametrize("form", ["host", "dev"])
def test_counts_under_contention(product_lib, form):
    """One pixel with 10^6 records and three with 10^5, shuffled into a random background: the warp-aggregated path."""
    b = _ctx(product_lib)
    rng = np.random.default_rng(21)
    bg = _records(_stream(200_000, 22))
    hot = np.concatenate([np.full(10**6, 5 + 7 * b.W), np.full(10**5, 100), np.full(10**5, 101), np.full(10**5, b.W * b.H - 1)])
    rec = np.concatenate([bg, np.repeat(bg[:1], hot.size)])
    rec["x"][bg.size:] = hot % b.W; rec["y"][bg.size:] = hot // b.W
    rec = rec[rng.permutation(rec.size)]
    _count(b, 0, rec, form, offset=5)
    c, _ = b.hotpix_read(0)
    ref = _bincount(rec, b.W, b.H)
    assert np.array_equal(c.ravel(), ref) and ref[5 + 7 * b.W] >= 10**6


def test_clear(product_lib):
    b = _ctx(product_lib)
    rec = _records(_stream(50_000, 23))
    hot = np.repeat(rec[:1], 20_000)
    rec = np.concatenate([rec, hot])
    _count(b, 0, rec)
    rc, n_hot = b.hotpix_select(0, 5)
    assert n_hot >= 1 and b.hotpix_read(0)[1].any()
    b.hotpix_clear(0)
    c, m = b.hotpix_read(0)
    assert not c.any() and not m.any()
    rec2 = _records(_stream(3000, 24))
    _count(b, 0, rec2, "dev", offset=3)
    assert np.array_equal(b.hotpix_read(0)[0].ravel(), _bincount(rec2, b.W, b.H))


# ---------------------------------------------------------------- selection
def _records_for_counts(c, W, seed):
    """Records (shuffled, ordered stamps) whose in-image counts are exactly c."""
    p = np.repeat(np.arange(c.size), c.astype(np.int64))
    p = p[np.random.default_rng(seed).permutation(p.size)]
    rec = np.zeros(p.size, rw.EVENT_DTYPE)
    rec["x"], rec["y"] = p % W, p // W
    t = T0 + np.arange(p.size, dtype=np.int64)
    rec["sec"], rec["nsec"] = t // 10**9, t % 10**9
    return rec


def _selection_cases(W, H):
    rng = np.random.default_rng(31)
    npix = W * H
    injected = rng.poisson(3.0, npix).astype(np.int64)
    injected[rng.choice(npix, 25, replace=False)] += rng.integers(40, 400, 25)
    return {"all-zero": np.zeros(npix, np.int64), "uniform": np.full(npix, 3, np.int64), "injected": injected,
            "sparse": np.where(rng.random(npix) < 0.01, rng.integers(1, 50, npix), 0)}


@pytest.mark.parametrize("case", ["all-zero", "uniform", "injected", "sparse"])
def test_mask_equals_rule(product_lib, case):
    b = _ctx(product_lib)
    c = _selection_cases(b.W, b.H)[case]
    if c.any():
        _count(b, 0, _records_for_counts(c, b.W, 32), "dev", offset=1)
    assert np.array_equal(b.hotpix_read(0)[0].ravel(), c.astype(np.uint64))
    for k in (0, 1, 5, 1e9):
        rc, n_hot = b.hotpix_select(0, k)
        m = b.hotpix_read(0)[1].ravel()
        ref = _rule(c, k)
        assert rc == 0 and np.array_equal(m, ref) and n_hot == int(ref.sum()), (case, k, n_hot, int(ref.sum()))
        if case in ("all-zero", "uniform"):
            assert n_hot == 0


def test_select_refuses_bad_k(product_lib):
    b = _ctx(product_lib)
    c = _selection_cases(b.W, b.H)["injected"]
    _count(b, 0, _records_for_counts(c, b.W, 33))
    b.hotpix_select(0, 5)
    m5 = b.hotpix_read(0)[1]
    for k in (-1.0, -1e-300, float("nan"), float("inf"), float("-inf")):
        rc, n_hot = b.hotpix_select(0, k, ok=(ERR_INVALID_ARG,))
        assert rc == ERR_INVALID_ARG and n_hot == -1, k
        assert np.array_equal(b.hotpix_read(0)[1], m5)


def test_count_past_u32_refused(product_lib):
    """One ~1 GB device buffer of 80 M identical records counted 53 times (4.24e9, fits u32) and then once more (past
    2^32 - 1): the selection refuses the counts and leaves the installed mask as it was; clear starts over."""
    import torch
    b = _ctx(product_lib)
    rec = np.zeros(1, rw.EVENT_DTYPE)
    rec["x"], rec["y"], rec["sec"] = 17, 9, 1_600_000_000
    n = 80_000_000
    buf = torch.from_numpy(np.frombuffer(rec.tobytes(), np.uint8).copy()).cuda().repeat(n)
    torch.cuda.synchronize()
    for _ in range(53):
        b.hotpix_count_event_array_dev(0, buf.data_ptr(), n)
    rc, n_hot = b.hotpix_select(0, 5)
    c, m = b.hotpix_read(0)
    assert rc == 0 and n_hot == 1 and int(c[9, 17]) == 53 * n and m[9, 17] == 1 and m.sum() == 1
    b.hotpix_count_event_array_dev(0, buf.data_ptr(), n)
    rc, _ = b.hotpix_select(0, 5, ok=(ERR_CAPACITY,))
    assert rc == ERR_CAPACITY
    assert np.array_equal(b.hotpix_read(0)[1], m)
    del buf
    b.hotpix_clear(0)
    rc, n_hot = b.hotpix_select(0, 5)
    assert rc == 0 and n_hot == 0 and not b.hotpix_read(0)[1].any()


# ---------------------------------------------------------------- masked pushes
HOT = [(5, 7), (100, 33), (345, 259), (0, 0), (200, 120), (17, 250)]


def _with_hot(rec, frac, seed, W):
    """A share frac of the records moved to the HOT pixels."""
    rec = rec.copy()
    rng = np.random.default_rng(seed)
    k = rng.random(rec.size) < frac
    h = rng.integers(0, len(HOT), int(k.sum()))
    rec["x"][k] = np.array([p[0] for p in HOT])[h]
    rec["y"][k] = np.array([p[1] for p in HOT])[h]
    return rec


class Masked:
    """A context with the HOT mask installed and one without a mask, fed the same records (the second prefiltered in numpy)."""

    def __init__(self, lib, form="host", ignore_polarity=0, rig="hkust"):
        self.m, self.u = _ctx(lib, rig, ignore_polarity), _ctx(lib, rig, ignore_polarity)
        self.form, self.W, self.H, self.k = form, self.m.W, self.m.H, 0
        c = np.zeros(self.W * self.H, np.int64)
        c[[y * self.W + x for x, y in HOT]] = 1000
        c[np.random.default_rng(41).choice(c.size, 3000, replace=False)] += 1
        for cam in (0, 1):
            _count(self.m, cam, _records_for_counts(c, self.W, 42))
            rc, n_hot = self.m.hotpix_select(cam, 5)
            m = self.m.hotpix_read(cam)[1].ravel()
            assert n_hot == len(HOT) and np.array_equal(np.flatnonzero(m), np.sort([y * self.W + x for x, y in HOT]))
        self.mask = m

    def keep(self, rec):
        x, y = rec["x"].astype(np.int64), rec["y"].astype(np.int64)
        inside = (x < self.W) & (y < self.H)
        hot = np.zeros(rec.size, bool)
        hot[inside] = self.mask[y[inside] * self.W + x[inside]] == 1
        return rec[~hot]

    def push(self, cam, rec, ok=(0,)):
        self.k += 1
        rc_m = _push(self.m, cam, rec, self.form, offset=self.k % 16, seed=self.k, ok=ok)
        rc_u = _push(self.u, cam, self.keep(rec), self.form, offset=(self.k + 5) % 16, seed=self.k, ok=ok)
        assert rc_m == rc_u and self.m.ts_events_pushed(cam) == self.u.ts_events_pushed(cam)
        return rc_m

    def same(self, cam, T):
        rm, im, mm = _build(self.m, cam, T)
        ru, iu, mu = _build(self.u, cam, T)
        assert rm == ru, (rm, ru, T)
        if rm == 0:
            assert im.tobytes() == iu.tobytes() and mm.tobytes() == mu.tobytes(), T
        return rm


@pytest.mark.parametrize("ignore_polarity", [0, 1])
@pytest.mark.parametrize("form", ["host", "dev"])
def test_masked_push_equals_prefiltered(product_lib, form, ignore_polarity):
    pr = Masked(product_lib, form, ignore_polarity)
    rec = _with_outside(_with_hot(_records(_stream(70_000, 43)), 0.3, 44, pr.W), pr.W, pr.H, 45)
    t = rec["sec"].astype(np.int64) * 10**9 + rec["nsec"]
    for cam in (0, 1):
        for a, z in ((0, 1), (1, 33), (33, 4096), (4096, 40_000), (40_000, 70_000)):
            pr.push(cam, rec[a:z])
            for T in (t[z - 1] + 1, t[(a + z) // 2], t[a]):
                assert pr.same(cam, T) == 0
        assert pr.m.ts_events_pushed(cam) == pr.keep(rec).size < rec.size


@pytest.mark.parametrize("where", ["hot", "kept"])
@pytest.mark.parametrize("form", ["host", "dev"])
def test_order_flag_after_the_filter(product_lib, form, where):
    """Stamps out of order only at hot pixels: the kept stream is ordered and the build succeeds.  Out of order at kept pixels
    (inside a push and at a push's first kept record): refused, as for the prefiltered push."""
    pr = Masked(product_lib, form)
    rec = _with_hot(_records(_stream(6000, 46)), 0.2, 47, pr.W)
    t = T0 + np.arange(rec.size, dtype=np.int64) * 1000
    hot = np.isin(rec["y"].astype(np.int64) * pr.W + rec["x"], [y * pr.W + x for x, y in HOT])
    pick = np.flatnonzero(hot if where == "hot" else ~hot)
    bad = pick[(pick > 100) & (pick < 5900)][::7]
    t[bad] -= 50_000                                     # older than its predecessors
    rec["sec"], rec["nsec"] = t // 10**9, t % 10**9
    pr.push(0, rec[:3000]); pr.push(0, rec[3000:])
    rc = pr.same(0, int(t.max()) + 1)
    assert rc == (0 if where == "hot" else ERR_UNSUPPORTED), (where, rc)


def test_unordered_mode_masked(product_lib):
    pr = Masked(product_lib, "host")
    rec = _with_hot(_records(_stream(20_000, 48)), 0.25, 49, pr.W)
    t = rec["sec"].astype(np.int64) * 10**9 + rec["nsec"] + np.random.default_rng(50).integers(-30_000, 30_000, rec.size)
    rec["sec"], rec["nsec"] = t // 10**9, t % 10**9
    for b in (pr.m, pr.u):
        b.ts_set_unordered_input(0, 1)
    for a, z in ((0, 1), (1, 4096), (4096, 20_000)):
        pr.push(0, rec[a:z])
        assert pr.same(0, int(t[:z].max()) + 1) == 0
    assert pr.same(0, int(np.median(t))) == 0


def test_event_windows_masked(product_lib):
    pr = Masked(product_lib, "dev")
    rec = _with_hot(_records(_stream(60_000, 51)), 0.3, 52, pr.W)
    for a, z in ((0, 10_000), (10_000, 35_000), (35_000, 60_000)):
        pr.push(0, rec[a:z])
    kt = pr.keep(rec)
    t = kt["sec"].astype(np.int64) * 10**9 + kt["nsec"]
    for b in (pr.m, pr.u):
        _build(b, 0, t[-1] + 1)
    for front, tb, te, budget, denoise in ((0, t[100], t[-1], 1000, 0), (0, t[20_000], t[-1], 1001, 1), (5000, t[0], t[30_000], 60_000, 0)):
        rm = pr.m.events_window_dev(0, front, tb, te, budget, denoise, 100_000)
        ru = pr.u.events_window_dev(0, front, tb, te, budget, denoise, 100_000)
        assert rm == ru
        for a, z in zip(pr.m.events_selected_dev(), pr.u.events_selected_dev()):
            assert np.array_equal(a, z)
    q = np.sort(np.concatenate([t[::997], t[::1999] + 1]))
    for k in range(0, q.size, 64):
        rm, i_m = pr.m.events_lower_bound_dev(0, 0, q[k:k + 64])
        ru, i_u = pr.u.events_lower_bound_dev(0, 0, q[k:k + 64])
        assert rm == ru == 0 and np.array_equal(i_m, i_u)


def test_fold_masked(product_lib):
    """7.5 M records (a fifth at hot pixels) in pushes of up to 1.5 M fold the kept log at the same points as the prefiltered
    pushes; builds at the newest stamp and refused builds inside the folded part agree after every push."""
    n = 7_500_000
    rng = np.random.default_rng(53)
    e = dict(x=rng.integers(0, 346, n).astype(np.uint16), y=rng.integers(0, 260, n).astype(np.uint16),
             t=(T0 + np.cumsum(rng.integers(0, 3, n))).astype(np.int64), p=rng.integers(0, 2, n).astype(np.uint8))
    pr = Masked(product_lib, "host")
    rec = _with_hot(_records(e), 0.2, 54, pr.W)
    cuts = [0, 1_500_000, 1_500_001, 3_000_000, 4_500_000, 6_000_000, n]
    refused = 0
    for a, z in zip(cuts[:-1], cuts[1:]):
        pr.push(0, rec[a:z])
        assert pr.same(0, e["t"][z - 1] + 1) == 0
        refused += pr.same(0, e["t"][max(0, z - 3_000_000)]) == ERR_UNSUPPORTED
    assert refused >= 1


@pytest.mark.parametrize("form", ["host", "dev"])
def test_push_of_hot_records_only(product_lib, form):
    pr = Masked(product_lib, form)
    rec = _records(_stream(5000, 55))
    pr.push(0, rec[:2000])
    before = pr.m.ts_events_pushed(0)
    hot = _with_hot(rec[2000:], 1.0, 56, pr.W)
    assert pr.keep(hot).size == 0
    pr.push(0, hot)
    assert pr.m.ts_events_pushed(0) == before
    assert pr.same(0, int(rec["sec"][1999]) * 10**9 + int(rec["nsec"][1999]) + 1) == 0
    pr.push(0, rec[2000:])
    assert pr.same(0, int(rec["sec"][-1]) * 10**9 + int(rec["nsec"][-1]) + 1) == 0


@pytest.mark.parametrize("form", ["host", "dev"])
def test_half_log_refusal_on_the_raw_count(product_lib, form):
    """A push of more than half the resident log is refused on the records handed in, even when fewer would be kept; it
    changes nothing.  Exactly half is taken."""
    pr = Masked(product_lib, form)
    small = _records(_stream(1000, 57))
    pr.push(0, small)
    big = _with_hot(_records(_stream(HALF_LOG + 1, 58, t0=T0 + 10**9)), 0.5, 59, pr.W)
    assert pr.keep(big).size <= HALF_LOG
    assert _push(pr.m, 0, big, form, offset=3, ok=(ERR_CAPACITY,)) == ERR_CAPACITY
    assert pr.m.ts_events_pushed(0) == pr.u.ts_events_pushed(0) == pr.keep(small).size
    t_small = int(small["sec"][-1]) * 10**9 + int(small["nsec"][-1])
    assert pr.same(0, t_small + 1) == 0
    pr.push(0, big[:HALF_LOG])
    assert pr.same(0, int(big["sec"][HALF_LOG - 1]) * 10**9 + int(big["nsec"][HALF_LOG - 1]) + 1) == 0


def test_reset_keeps_the_mask(product_lib):
    pr = Masked(product_lib, "host")
    rec = _with_hot(_records(_stream(8000, 60)), 0.3, 61, pr.W)
    pr.push(0, rec)
    for b in (pr.m, pr.u):
        b.ts_reset(0)
    assert pr.m.hotpix_read(0)[1].sum() == len(HOT)
    pr.push(0, rec)
    assert pr.same(0, int(rec["sec"][-1]) * 10**9 + int(rec["nsec"][-1]) + 1) == 0


# ---------------------------------------------------------------- end to end: bag_system --hot-pixels
N_HOT = 20
# 500 Hz - 5 kHz: over the 1.3 s scenes a 100 Hz pixel has 130 events, below mu + 5 sigma (about 200 to 250 with the faster
# injected pixels in the statistic), so the slowest injected rate is 500 Hz (650 events).
HOT_RATES = np.geomspace(500.0, 5000.0, N_HOT)


def _inject(e, pix, W, seed):
    """e plus N_HOT pixels firing at HOT_RATES over e's time span, merged by stamp (stable: e's order is kept)."""
    rng = np.random.default_rng(seed)
    t0, t1 = int(e["t"][0]), int(e["t"][-1])
    xs, ys, ts, ps = [e["x"]], [e["y"]], [e["t"]], [e["p"]]
    for p, rate in zip(pix, HOT_RATES):
        period = int(round(1e9 / rate))
        t = np.arange(t0 + int(rng.integers(0, period)), t1, period, dtype=np.int64)
        xs.append(np.full(t.size, p % W, np.uint16)); ys.append(np.full(t.size, p // W, np.uint16))
        ts.append(t); ps.append(rng.integers(0, 2, t.size).astype(np.uint8))
    t = np.concatenate(ts)
    o = np.argsort(t, kind="stable")
    return dict(x=np.concatenate(xs)[o], y=np.concatenate(ys)[o], t=t[o], p=np.concatenate(ps)[o])


@pytest.mark.parametrize("scene", ["dense", "mapping"])
def test_bag_system_hot_pixels_equals_system_loop_prefiltered(product_lib, tmp_path, scene):
    """The scenes of tests/test_system_loop.py with 20 hot pixels per camera (different ones left and right) written into a
    bag: the rule selects exactly the injected pixels, on the device as in numpy, and bag_system --hot-pixels 5 gives the tick
    records, trajectory file and final map of system_loop on the streams without the events at those pixels, byte for byte."""
    import indep_system as isy
    from esvo_b200 import configs
    import test_system_loop as tsl
    s = tsl._stream(scene)
    t0, n = tsl._ticks(s)
    W, H = 346, 260
    rng = np.random.default_rng(62)
    pix = rng.choice(W * H, 2 * N_HOT, replace=False)
    dirty = {"left": _inject(s["left"], pix[:N_HOT], W, 63), "right": _inject(s["right"], pix[N_HOT:], W, 64)}
    b = _ctx(product_lib)
    clean = {}
    for cam, side, hot in ((0, "left", pix[:N_HOT]), (1, "right", pix[N_HOT:])):
        e = dirty[side]
        rec = _records(e)
        c = _bincount(rec, W, H)
        ref = _rule(c, 5)
        assert np.array_equal(np.flatnonzero(ref), np.sort(hot)), side
        b.hotpix_count_event_array(cam, [rec.tobytes()])
        rc, n_hot = b.hotpix_select(cam, 5)
        assert n_hot == N_HOT and np.array_equal(b.hotpix_read(cam)[1].ravel(), ref)
        keep = ref[e["y"].astype(np.int64) * W + e["x"]] == 0          # every record of the scenes is inside the image
        clean[side] = {k: v[keep] for k, v in e.items()}
    b.close()
    scen, res_a, traj_a = tmp_path / "scen.bin", tmp_path / "a.bin", tmp_path / "a.txt"
    isy.write_scenario(scen, W, H, t0, tsl.DT_NS, n, clean["left"], clean["right"])
    p = subprocess.run([_compile(tmp_path, "system_loop"), str(scen), str(res_a), str(traj_a)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    rr = configs.RIGS["hkust"]
    L, R, LI, RI = "/davis/left/events", "/davis/right/events", "/davis/left/camera_info", "/davis/right/camera_info"
    infos = {t: (rr["width"], rr["height"], rr["model"], rr[sd]["D"], rr[sd]["K"], rr[sd]["R"], rr[sd]["P"]) for t, sd in ((LI, "left"), (RI, "right"))}
    bag = tmp_path / "scene.bag"
    rw.write_event_bag(bag, {L: dirty["left"], R: dirty["right"]}, infos=infos, msg_events=1500, chunk_threshold=64 * 1024)
    res_b, traj_b = tmp_path / "b.bin", tmp_path / "b.txt"
    p = subprocess.run([_compile(tmp_path, "bag_system"), str(bag), L, R, LI, RI, str(res_b), str(traj_b), "--t0-ns", str(t0),
                        "--dt-ns", str(tsl.DT_NS), "--ticks", str(n), "--hot-pixels", "5"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    assert f"hot pixels left: {N_HOT}" in p.stdout and f"hot pixels right: {N_HOT}" in p.stdout, p.stdout
    a, bb = isy.parse_result(res_a), isy.parse_result(res_b)
    assert a[0].size == bb[0].size == n and a[3] == bb[3] == 0
    for k in ["t", "status", "has_pose", "T"]:
        assert a[0][k].tobytes() == bb[0][k].tobytes(), k
    assert a[1].tobytes() == bb[1].tobytes() and a[2].tobytes() == bb[2].tobytes()
    assert traj_a.read_bytes() == traj_b.read_bytes() and len(traj_a.read_bytes()) > 0
