"""Case table of the event-to-event matcher (esvo_em_match) beyond the shipped configuration, shared by tests/test_em_pins.py
(the oracle against tests/indep_numpy.py::event_match, no GPU) and tests/test_gpu_em_parity.py (the device against the
oracle, bit for bit).

Every case is built deterministically here: its own rectification LUTs (set through esvo_set_rectify_tables on both sides),
time-surface pair, left / right events, slices and poses.  Observation and slice poses are translations with dyadic entries,
so rigid_inverse(T_obs) * T_slice is exact and T_left_rv = I wherever a slice sits at the observation pose.

LUT kinds: "int" -- both LUTs map a raw pixel onto itself, so with T_left_rv = I every warp lands exactly on a pixel
boundary and the last bit of cam2World decides floor(x1) and the border tests ("boundary" cases: device against oracle
only; the numpy path inverts with np.linalg.inv, a third rounding); "quarter" -- (x + 1/4, y + 1/4), where no decision sits
within rounding of a boundary; "rig" -- the rig's own tables (esvo_compute_rectify_tables).  Time surfaces: a smooth
texture on the left and the same texture shifted by TRUE_D pixels on the right, so the candidate at disparity TRUE_D
scores near 0; "zero-left" makes every scored candidate cost exactly 0.5."""
import functools

import numpy as np

import indep_numpy as ind
from esvo_b200 import capi, configs
from util import TS_EPOCH, build_ts_pair, em_problem, scenario

T_SMALL = 1_000_000_000                    # 1 s
T_OBS = (0.25, -0.5, 0.125)                # observation pose: a dyadic translation
TRUE_D = 4                                 # disparity of the textured pair
SHIPPED = dict(time_thr=5e-4, epi_thr=1.0, ncc_thr=0.1)   # EM_Time_THRESHOLD, EM_EPIPOLAR_THRESHOLD, EM_TS_NCC_THRESHOLD
GAP_NS = 10_000_000                        # left events 10 ms apart: their time windows never overlap


def pose(t=(0.0, 0.0, 0.0)):
    T = np.eye(4)
    T[:3, 3] = np.add(T_OBS, t)
    return T


def texture(W, H, seed=0):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    v = np.zeros((H, W))
    for _ in range(6):
        kx, ky, ph = rng.uniform(0.08, 0.45), rng.uniform(-0.45, 0.45), rng.uniform(0, 2 * np.pi)
        v += np.sin(kx * x + ky * y + ph)
    v = (v - v.min()) / (v.max() - v.min())
    return np.rint(255 * v).astype(np.uint8)


def ts_pair(W, H, kind="texture", seed=0):
    t = texture(W + TRUE_D, H, seed)
    tl, tr = t[:, :W].copy(), t[:, TRUE_D:].copy()          # tr[y, x] = tl[y, x + TRUE_D]
    if kind == "zero-left":
        tl[:] = 0
    return tl, tr


def grid_lut(W, H, off):
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    return np.stack([x + off, y + off], axis=-1)


@functools.lru_cache(maxsize=None)
def rig_luts(rig):
    """The rig's own LUTs, from the product's context-free table builder (pinned to cv2 in test_product_tables_cv2.py)."""
    lib = capi.load_product()
    return tuple(capi.compute_rectify_tables(lib, c)[2] for c in configs.rig_calibs(rig))


def rig_size(rig):
    r = configs.RIGS[rig]
    return r["width"], r["height"]


class _Ev:
    """Left events with their own candidates; right events come out time-ordered (stable on equal stamps)."""

    def __init__(self):
        self.left, self.right = [], []

    def add(self, x, y, t, p=1):
        self.left.append((x, y, t, p))

    def cand(self, x, y, t, p=1):
        self.right.append((x, y, t, p))

    def arrays(self):
        def pack(rows, order=None):
            a = np.array(rows, np.int64).reshape(-1, 4)
            if order is not None:
                a = a[order]
            return dict(x=a[:, 0].astype(np.uint16), y=a[:, 1].astype(np.uint16), t=a[:, 2].copy(), p=a[:, 3].astype(np.uint8))
        rt = np.array([r[2] for r in self.right], np.int64)
        return pack(self.left), pack(self.right, np.argsort(rt, kind="stable"))


def _case(id, build, boundary=False, **kw):
    return dict(id=id, build=build, boundary=boundary, kw=kw)


def _inputs(rig, lut, ts, ev, slices=None, poses=None, T_obs=None):
    W, H = rig_size(rig)
    if lut == "rig":
        lut_l, lut_r = rig_luts(rig)
    elif isinstance(lut, tuple):
        lut_l, lut_r = lut
    else:
        lut_l = lut_r = grid_lut(W, H, {"int": 0.0, "quarter": 0.25}[lut])
    tl, tr = ts if isinstance(ts, tuple) else ts_pair(W, H, ts)
    left, right = ev.arrays()
    n = left["x"].size
    counts = np.array([n] if slices is None else slices, np.int32)
    if poses is None:
        poses = [pose() for _ in counts]
    return dict(rig=rig, lut_l=np.ascontiguousarray(lut_l), lut_r=np.ascontiguousarray(lut_r), tl=tl, tr=tr,
                T_obs=pose() if T_obs is None else T_obs, left=left, right=right, counts=counts,
                poses=np.array([np.asarray(P, float).ravel() for P in poses]))


# ---- integer / quarter-pixel rigs: left events on every border of the warp and the patch test --------------------------
def _borders(W, H, wx, wy):
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    xs = sorted({v for v in (hx - 1, hx, hx + 1, hx + 2, W // 2, W - hx - 3, W - hx - 2, W - hx - 1, W - hx, W - 1) if 0 <= v < W})
    ys = sorted({v for v in (hy - 1, hy, hy + 1, H // 2, H - hy - 2, H - hy - 1, H - hy, H - 1) if 0 <= v < H})
    return xs, ys


def b_borders(rig, lut, wx, wy, moving=False):
    def build():
        W, H = rig_size(rig)
        ev = _Ev()
        xs, ys = _borders(W, H, wx, wy)
        t = T_SMALL
        for y in ys:
            for x in xs:
                ev.add(x, y, t)
                for k, d in enumerate((1, 2, 3, TRUE_D, 6, 9)):
                    if x - d >= 0:
                        ev.cand(x - d, y, t - 20_000 + 1_000 * k)
                t += GAP_NS
        n = len(ev.left)
        if not moving:
            return _inputs(rig, lut, "texture", ev)
        half = n // 2
        return _inputs(rig, lut, "texture", ev, slices=[half, n - half], poses=[pose((0.015625, 0.0, 0.0)), pose((0.0, 0.0078125, -0.03125))])
    return build


# ---- exact ties: a left time surface of zeros scores every candidate 0.5 -------------------------------------------------
TIE_KS = (0, 5, 31, 32, 33, 70)
TIE_X, TIE_Y = 60, 100


def tie_layout():
    """(k, number of candidates) per left event: the first k fail the warp (x2 < hx), the rest score exactly 0.5."""
    return [(k, max(40, min(100, k + 30))) for k in TIE_KS]


def b_ties():
    W, H = rig_size("hkust")
    ev = _Ev()
    t = T_SMALL
    for k, n in tie_layout():
        ev.add(TIE_X, TIE_Y, t)
        for q in range(n):
            d = TIE_X - 1 if q < k else 1 + q % 30            # x2 = 1.25 < hx: warping2 rejects it
            ev.cand(TIE_X - d, TIE_Y, t - 40_000 + 500 * q)
        t += GAP_NS
    return _inputs("hkust", "quarter", "zero-left", ev)


# ---- no candidate scores: every epipolar survivor fails the warp, behind candidates that fail the epipolar test ---------
def b_fallback():
    ev = _Ev()
    t = T_SMALL
    for x in (40, 120, 200, 300):
        ev.add(x, 130, t)
        for q in range(3):
            ev.cand(x - 5 - q, 134, t - 30_000 + 1_000 * q)     # 4 rows away: epipolar reject
        for q in range(4):
            ev.cand(1 + q, 130, t - 20_000 + 1_000 * q)         # x2 < hx: warp reject
        t += GAP_NS
    return _inputs("hkust", "quarter", "texture", ev)


# ---- epipolar boundaries and left LUT entries off the image ---------------------------------------------------------------
EPI_THR = 0.5


def b_epi():
    """Rows near 0 (patch height 1): LUT rows below 1 resolve |dy| to 1.1e-16.  Per left event one candidate, so ncc 1 shows
    whether the epipolar test let it through (accepted, scored or by the fallback) or not (no seed)."""
    W, H = rig_size("hkust")
    lut_l, lut_r = grid_lut(W, H, 0.25), grid_lut(W, H, 0.25)
    xl1 = 0.75
    up = np.nextafter(EPI_THR, np.inf)
    rows = [xl1 - EPI_THR, xl1 + EPI_THR, xl1 - up, np.nextafter(xl1 + EPI_THR, np.inf)]   # |dy|: thr, thr, next above, 2 ulp above
    ev = _Ev()
    t = T_SMALL
    specs = []                                                  # (left LUT (x, y), right LUT (x, y))
    for r in rows:
        specs.append(((100.25, xl1), (95.25, r)))
    specs.append(((150.25, xl1), (150.25, xl1)))                # xr0 == xl0: rejected
    specs.append(((160.25, xl1), (np.nextafter(160.25, -np.inf), xl1)))   # one ulp of disparity: accepted, huge finite depth
    specs.append(((-3.25, xl1), (-9.25, xl1)))                  # left LUT off the image (negative)
    specs.append(((W + 2.75, xl1), (W - 3.25, xl1)))            # ... and beyond W
    for k, (l, r) in enumerate(specs):
        lx, rx = 10 + k, 10 + k                                 # raw pixels on rows 200 / 201 carry the hand-set entries
        lut_l[200, lx] = l
        lut_r[201, rx] = r
        ev.add(lx, 200, t)
        ev.cand(rx, 201, t + 1_000)
        ev.cand(rx, 202, t + 2_000)                             # an ordinary entry 201 rows away: always an epipolar reject
        t += GAP_NS
    assert [abs(xl1 - r) for r in rows] == [EPI_THR, EPI_THR, up, np.nextafter(up, np.inf)]
    return _inputs("hkust", (lut_l, lut_r), "texture", ev)


# ---- time windows: candidates on the bounds of ros::Time(toSec() -/+ thr / 2), small and epoch stamps -----------------
def window_bounds(te, thr):
    tes = ind.ros_to_sec(te)
    return ind.ros_from_sec(tes - thr / 2), ind.ros_from_sec(tes + thr / 2)


def b_windows(t0, thr):
    def build():
        ev = _Ev()
        t = t0
        for i, x in enumerate((60, 110, 160, 210, 260)):
            ev.add(x, 90 + 20 * i, t, i % 2)
            lo, hi = window_bounds(t, thr)
            offs = [lo - 300, lo - 1, lo, lo + 1, lo + 300, t, hi - 300, hi - 1, hi, hi + 1, hi + 300]
            for q, s in enumerate(offs):
                d = 1 + (q * 3 + i) % 9
                ev.cand(x - d, 90 + 20 * i, s, i % 2)
                ev.cand(x - d - 1, 90 + 20 * i, s, 1 - i % 2)   # the other polarity on the same stamp
            t += GAP_NS
        return _inputs("hkust", "quarter", "texture", ev)
    return build


def b_equal_runs(t0, thr):
    """Runs of equal stamps, both polarities, on each side of both window bounds.  At time_thr = 0 the window
    [lower_bound(low), lower_bound(up)) is empty: nothing matches, nothing is scored."""
    def build():
        ev = _Ev()
        t = t0
        for i, x in enumerate((80, 180, 280)):
            ev.add(x, 120, t, 1)
            lo, hi = window_bounds(t, thr)
            for q, s in enumerate((lo - 1, lo - 1, lo, lo, lo, lo + 1, t, t, hi - 1, hi - 1, hi, hi, hi + 1, hi + 1)):
                for p in (0, 1):
                    ev.cand(x - 1 - (q + i) % 8, 120, s, p)
            t += GAP_NS + 137
        return _inputs("hkust", "quarter", "texture", ev)
    return build


def b_natural_epoch(rig, n_left):
    """The natural scenario (tests/util.py::scenario, em_problem) with every stamp shifted to the UNIX epoch."""
    def build(oracle_be_for):
        s = scenario(rig, seed=4, n_seeds=800, t_ts=0.5)
        be = oracle_be_for(rig)
        tl, tr = build_ts_pair(be, s)
        be.ts_reset(0); be.ts_reset(1)
        left, right, counts, poses = em_problem(s, max_events=n_left)
        shift = TS_EPOCH - (TS_EPOCH % 1_000_000_000)
        for e in (left, right):
            e["t"] = e["t"] + shift
        lut_l, lut_r = rig_luts(rig)
        return dict(rig=rig, lut_l=lut_l, lut_r=lut_r, tl=tl, tr=tr, T_obs=np.asarray(s["T_world_left"], float).reshape(4, 4),
                    left=left, right=right, counts=counts, poses=poses)
    build.needs_backend = True
    return build


# ---- crowded windows: > 32 and > 1 000 right candidates per left event -------------------------------------------------
def b_crowd(n_cand, n_left):
    def build():
        W, H = rig_size("hkust")
        rng = np.random.default_rng(n_cand)
        ev = _Ev()
        t = T_SMALL
        xs = rng.integers(40, W - 20, n_left)
        for i in range(n_left):
            ev.add(int(xs[i]), 60 + 4 * i, t + i)              # every left event sees the same window
        for q in range(n_cand):
            i = q % n_left
            x, y = int(xs[i]), 60 + 4 * i
            kind = q % 5
            if kind == 0:                                       # epipolar survivor at a varying disparity
                ev.cand(x - 1 - (q // 5) % 12, y, t - 40_000 + 60 * q % 80_000)
            elif kind == 1:
                ev.cand(x - 2, y, t - 40_000 + 60 * q % 80_000, 0)   # wrong polarity
            else:
                ev.cand(int(rng.integers(0, W)), int(rng.integers(0, H)), t - 40_000 + 60 * q % 80_000)
        return _inputs("hkust", "quarter", "texture", ev)
    return build


# ---- random interior scenes: patch shapes, thread orders, slicing, rigs -------------------------------------------------
def b_random(n_left, rig="hkust", lut="quarter", seed=0, slices=None, n_cand=6):
    def build():
        W, H = rig_size(rig)
        rng = np.random.default_rng(seed)
        ev = _Ev()
        t = T_SMALL
        for i in range(n_left):
            x, y = int(rng.integers(12, W - 2)), int(rng.integers(1, H - 1))
            p = int(rng.integers(0, 2))
            ev.add(x, y, t, p)
            for q in range(n_cand):
                d = TRUE_D if q == 2 else int(rng.integers(1, 12))
                yr = min(max(y + int(rng.integers(-1, 2)), 0), H - 1) if lut == "rig" else y
                ev.cand(max(x - d, 0), yr, t + int(rng.integers(-40_000, 40_000)), p if q % 4 else 1 - p)
            t += 100_000
        n = len(ev.left)
        sl = [n // 3, n // 3, n - 2 * (n // 3)] if slices is None else slices
        offs = [(0.0, 0.0, 0.0), (0.015625, -0.0078125, 0.0), (-0.03125, 0.0, 0.0625)]
        poses = [pose(offs[k % 3]) for k in range(len(sl))]
        return _inputs(rig, lut, "texture", ev, slices=sl, poses=poses)
    return build


CASES = [
    # integer rig, T_left_rv = I: every warp on a pixel boundary (device against oracle only)
    _case("int-borders-15x7", b_borders("hkust", "int", 15, 7), True, patch=(15, 7), ncc_thr=1.0),
    _case("int-borders-16x6", b_borders("hkust", "int", 16, 6), True, patch=(16, 6), ncc_thr=1.0),
    _case("int-borders-2x2", b_borders("hkust", "int", 2, 2), True, patch=(2, 2), ncc_thr=1.0),
    _case("int-borders-1x15", b_borders("hkust", "int", 1, 15), True, patch=(1, 15), ncc_thr=1.0),
    _case("int-borders-25x5-dsec", b_borders("dsec", "int", 25, 5), True, patch=(25, 5), ncc_thr=0.3),
    # the quarter-pixel twins
    _case("q-borders-15x7", b_borders("hkust", "quarter", 15, 7), patch=(15, 7), ncc_thr=1.0),
    _case("q-borders-16x6", b_borders("hkust", "quarter", 16, 6), patch=(16, 6), ncc_thr=1.0),
    _case("q-borders-2x2-moving", b_borders("hkust", "quarter", 2, 2, moving=True), patch=(2, 2), ncc_thr=0.5),
    # exact ties
    _case("ties-ncc0.5", b_ties, patch=(15, 7), ncc_thr=0.5, num_thread=3),
    _case("ties-ncc1", b_ties, patch=(15, 7), ncc_thr=1.0, num_thread=1),
    # no candidate scores
    _case("fallback-ncc1", b_fallback, patch=(15, 7), ncc_thr=1.0),
    _case("fallback-ncc0.99", b_fallback, patch=(15, 7), ncc_thr=0.99),
    # epipolar bounds, off-image left entries
    _case("epi-bounds", b_epi, patch=(15, 1), epi_thr=EPI_THR, ncc_thr=1.0, num_thread=2),
    # time windows
    _case("win-small", b_windows(T_SMALL, 1e-4), time_thr=1e-4, ncc_thr=1.0, patch=(15, 7)),
    _case("win-epoch", b_windows(TS_EPOCH, 1e-4), time_thr=1e-4, ncc_thr=1.0, patch=(15, 7)),
    _case("win-epoch-shipped", b_windows(TS_EPOCH + 123_456_789, 5e-4), time_thr=5e-4, ncc_thr=1.0, patch=(25, 5)),
    _case("win-equal-runs-small", b_equal_runs(T_SMALL, 2e-6), time_thr=2e-6, ncc_thr=1.0, patch=(15, 7)),
    _case("win-equal-runs-epoch", b_equal_runs(TS_EPOCH + 1, 2e-6), time_thr=2e-6, ncc_thr=1.0, patch=(15, 7)),
    _case("win-zero-thr-small", b_equal_runs(T_SMALL, 0.0), time_thr=0.0, ncc_thr=1.0, patch=(15, 7)),
    _case("win-zero-thr-epoch", b_equal_runs(TS_EPOCH + 1, 0.0), time_thr=0.0, ncc_thr=1.0, patch=(15, 7)),
    _case("natural-epoch-hkust", b_natural_epoch("hkust", 300), patch=(25, 5), num_thread=4, **SHIPPED),
    _case("natural-epoch-dsec", b_natural_epoch("dsec", 300), patch=(15, 7), num_thread=4, **SHIPPED),
    # crowded windows
    _case("crowd-40", b_crowd(40 * 6, 6), ncc_thr=0.3, patch=(15, 7)),
    _case("crowd-1200", b_crowd(1200 * 4, 4), ncc_thr=0.3, patch=(15, 7)),
    # patch shapes
    *[_case(f"shape-{wx}x{wy}", b_random(60, seed=wx * 100 + wy), patch=(wx, wy),
            ncc_thr=0.5 if wx * wy == 1 else 0.3)                     # a 1x1 patch is constant: every score is exactly 0.5
      for wx, wy in ((1, 1), (2, 2), (16, 6), (1, 15), (15, 1), (31, 3), (25, 5))],
    _case("shape-176x3", b_random(60, seed=5), patch=(176, 3), ncc_thr=0.3),        # wider than half the image
    _case("shape-wider-than-image", b_random(40, seed=5), patch=(349, 3), ncc_thr=0.3),   # hx > W - hx: every warp fails
    # thread order and slicing: event totals 1, 31, 256, 257, 513; NT 1, 2, 7, 256, > total
    _case("nt1-total1", b_random(1, seed=11), num_thread=1, ncc_thr=1.0),
    _case("nt4-total1", b_random(1, seed=11), num_thread=4, ncc_thr=1.0),
    _case("nt7-total31", b_random(31, seed=12), num_thread=7, ncc_thr=0.5),
    _case("nt256-total256", b_random(256, seed=13, n_cand=3), num_thread=256, ncc_thr=0.5),
    _case("nt2-total257", b_random(257, seed=14, n_cand=3), num_thread=2, ncc_thr=0.5),
    _case("nt300-total257", b_random(257, seed=14, n_cand=3), num_thread=300, ncc_thr=0.5),
    _case("nt7-total513", b_random(513, seed=15, n_cand=2), num_thread=7, ncc_thr=0.5),
    _case("slices-zero-neg-below", b_random(120, seed=16, slices=[20, 0, -7, 30, 0, 25]), num_thread=3, ncc_thr=0.5),
    _case("slices-neg-above", b_random(120, seed=17, slices=[-3, 70, 0, 90]), num_thread=5, ncc_thr=0.5),
    # rigs, on their own tables
    *[_case(f"rig-{r}", b_random(150, rig=r, lut="rig", seed=20 + k, n_cand=8), ncc_thr=0.6, epi_thr=1.0, num_thread=4)
      for k, r in enumerate(("hkust", "dsec", "rpg", "upenn"))],
]
CASES = {c["id"]: c for c in CASES}


def params(rig, lib):
    return configs.params_for(rig, lib) if rig in ("hkust", "dsec") else configs.mvstereo_params_for(rig, lib)


def case_kw(c):
    kw = dict(time_thr=5e-4, epi_thr=1.0, ncc_thr=0.1, patch=(15, 7), num_thread=4)
    kw.update(c["kw"])
    return kw


def case_inputs(c, oracle_be_for=None):
    """The inputs of case c; oracle_be_for(rig) supplies an oracle backend where a case builds its time surfaces on one."""
    b = c["build"]
    return b(oracle_be_for) if getattr(b, "needs_backend", False) else b()


def load_case(be, inp):
    """Hands a context of the case's rig the case's LUTs and observation pair; returns it."""
    for cam, lut in ((0, inp["lut_l"]), (1, inp["lut_r"])):
        be.set_rectify_tables(cam, lut=np.asarray(lut, np.float64).reshape(be.H, be.W, 2))
    be.set_ts_pair(inp["tl"], inp["tr"], inp["T_obs"])
    return be


def run(be, inp, kw):
    return be.em_match(inp["left"], inp["right"], inp["counts"], inp["poses"], **kw)


def numpy_match(inp, kw, baseline, info=None):
    cams = configs.rig_arrays(inp["rig"])
    P = cams["left"]["P"], cams["right"]["P"]
    return ind.event_match(inp["left"], inp["right"], inp["counts"], inp["poses"], inp["lut_l"], inp["lut_r"], P[0], P[1], baseline,
                           inp["tl"], inp["tr"], inp["T_obs"], kw["time_thr"], kw["epi_thr"], kw["ncc_thr"], kw["patch"][0],
                           kw["patch"][1], kw["num_thread"], info=info)


def em_match_raw(be, inp, kw, capacity, with_buffer=True):
    """esvo_em_match / esvo_oracle_em_match through ctypes with a chosen capacity: (status, *n_seeds, *n_patch_evals)."""
    import ctypes as C
    prm = capi.EmParams(kw["time_thr"], kw["epi_thr"], kw["ncc_thr"], kw["patch"][0], kw["patch"][1], kw["num_thread"], 0)

    def ev(d):
        return [np.ascontiguousarray(d[k], t) for k, t in (("x", np.uint16), ("y", np.uint16), ("t", np.int64), ("p", np.uint8))]
    L, R = ev(inp["left"]), ev(inp["right"])
    sc = np.ascontiguousarray(inp["counts"], np.int32); sp = np.ascontiguousarray(inp["poses"], np.float64)
    out = np.zeros(max(capacity, 1), capi.SEED_DTYPE) if with_buffer else None
    n = C.c_size_t(capacity); evals = C.c_uint64(0)
    ct = (C.c_uint16, C.c_uint16, C.c_int64, C.c_uint8)
    E = [C.POINTER(t) for t in ct] + [C.c_size_t]
    rc = be._call("em_match", [C.POINTER(capi.EmParams)] + E + [C.POINTER(C.c_int32), C.POINTER(C.c_double), C.c_size_t] + E +
                  [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)],
                  C.byref(prm), *[a.ctypes.data_as(C.POINTER(t)) for a, t in zip(L, ct)], L[0].size,
                  sc.ctypes.data_as(C.POINTER(C.c_int32)), sp.ctypes.data_as(C.POINTER(C.c_double)), sc.size,
                  *[a.ctypes.data_as(C.POINTER(t)) for a, t in zip(R, ct)], R[0].size,
                  None if out is None else out.ctypes.data_as(C.c_void_p), C.byref(n), C.byref(evals), ok=(0, -4))
    return rc, n.value, evals.value
