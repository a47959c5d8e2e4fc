"""Shared helpers for the parity tests: one synthetic scenario, two backends fed identical inputs."""
import ctypes as C
import functools

import numpy as np

from esvo_b200 import capi, configs, synth


@functools.lru_cache(maxsize=8)
def scenario(rig="hkust", seed=2, n_seeds=1500, t_ts=0.5):
    kw = {}
    if rig == "dsec":
        kw = dict(n_segments=120)
    return synth.make_stream(rig, seed=seed, n_seeds=n_seeds, t_ts=t_ts, **kw)


def make_backends(rig, oracle_lib, product_lib, tweak=None):
    l, r = configs.rig_calibs(rig)
    po = configs.params_for(rig, oracle_lib)
    pp = configs.params_for(rig, product_lib)
    if tweak:
        tweak(po); tweak(pp)
    o = capi.Backend(oracle_lib, l, r, po)
    g = capi.Backend(product_lib, l, r, pp)
    # The product runs on ITS OWN rectification tables (host_setup.cpp, pinned to cv2 bit for bit in
    # tests/test_product_tables_cv2.py); the checker gets the same tables so that both sides see identical inputs.
    for cam in (0, 1):
        m1, m2, lut, mask = g.get_rectify_tables(cam)
        o.set_rectify_tables(cam, m1, m2, lut, mask)
    return o, g


def build_ts_pair(b, s):
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        b.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
    _, tl = b.ts_build(0, s["t_ts_ns"], want_idx=False)
    _, tr = b.ts_build(1, s["t_ts_ns"], want_idx=False)
    return tl, tr


def rel(a, b):
    a = np.asarray(a, float); b = np.asarray(b, float)
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-300)


# Contributions per pixel of fold_vector: around every bound of the fold kernel's list handling (register networks of 32 / 64,
# three merged runs up to 192, the sort pool beyond, the 255 length bin of the list-length sort).
FOLD_LENGTHS = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 500)


def fold_vector(Pl, lengths=FOLD_LENGTHS, seed=0, td_nu=2.1897):
    """A hand-built point vector that puts lists of exactly `lengths` contributions on separate pixels of a 346 x 260 map
    (observation and frame poses are the identity, each point projects inside its target pixel; targets are 45 / 55 px
    apart, so the 2 x 2 / 3 x 3 splats of fusion radius 0 / 1 and of the naive propagation never meet).  The points of all
    pixels are interleaved.  Inverse depths alternate at random between two clusters (1.0 and 0.5) and standard deviations
    spread over 0.005 .. 0.3, so that create, compatible fuse, occlusion skip and replace all happen and the surviving
    element depends on the order of the replay.  Returns (points, [(row, col, length)])."""
    import indep_numpy as ind
    rng = np.random.default_rng(seed)
    recs, targets = [], []
    for i, L in enumerate(lengths):
        row, col = 20 + 45 * (i // 6), 25 + 55 * (i % 6)
        targets.append((row, col, L))
        for _ in range(L):
            rho = (0.5 if rng.random() < 0.5 else 1.0) * (1 + 0.02 * rng.standard_normal())
            var = (10 ** rng.uniform(-2.3, -0.5)) ** 2
            x = np.array([col + rng.uniform(0.2, 0.8), row + rng.uniform(0.2, 0.8)])
            recs.append((row, col, x, rho, var, rng.uniform(1, 100), int(rng.integers(0, 4))))
    pts = np.zeros(len(recs), capi.DEPTH_POINT_DTYPE)
    for k, j in enumerate(rng.permutation(len(recs))):
        row, col, x, rho, var, res, age = recs[j]
        q = pts[k]
        q["row"], q["col"], q["x"], q["inv_depth"] = row, col, x, rho
        q["nu"], q["variance"], q["scale2"] = td_nu, var, var * (td_nu - 2) / td_nu
        q["residual"], q["age"] = res, age
        q["p_cam"] = ind.cam2world(Pl, x, rho)
        q["T_world_cam"] = np.eye(4).ravel()
    return pts, targets


def fold_replay(pts, Pl, W, H, radius, naive=False, stats=None):
    """tests/indep_fusion.py replay of one vector into an empty map: (grid, number of fusions).  stats (dict, optional)
    receives the number of times each branch of the case analysis was taken."""
    import indep_fusion as inf
    grid = inf.Grid(H, W)
    vec = [dict(p_cam=q["p_cam"], s2=float(q["scale2"]), nu=float(q["nu"]), var=float(q["variance"]), res=float(q["residual"]),
                age=int(q["age"]), T_world_cam=q["T_world_cam"]) for q in pts]
    if naive:
        inf.naive_propagate_vector(grid, vec, np.eye(4), Pl, W, H, stats)
        return grid, 0
    return grid, inf.fuse_vector(grid, vec, np.eye(4), Pl, W, H, radius, stats)


def grid_vs_map(grid, m, tag, rtol=1e-10):
    """An indep_fusion grid against a downloaded map: element order, ages exact; values within rtol."""
    assert len(grid.elements) == m.size, (tag, len(grid.elements), m.size)
    assert [e.row for e in grid.elements] == m["row"].tolist() and [e.col for e in grid.elements] == m["col"].tolist(), tag + ": element order"
    assert [e.age for e in grid.elements] == m["age"].tolist(), tag + ": ages"
    for name, get in (("inv_depth", lambda e: e.rho), ("scale2", lambda e: e.s2), ("nu", lambda e: e.nu), ("variance", lambda e: e.var),
                      ("residual", lambda e: e.res)):
        a = np.array([get(e) for e in grid.elements]); b = m[name]
        assert np.allclose(a, b, rtol=rtol, atol=1e-300), (tag, name, np.abs(a - b).max())
    pc = np.array([e.p_cam for e in grid.elements])
    assert np.allclose(pc, m["p_cam"], rtol=1e-9, atol=1e-12), tag + ": p_cam"
    xx = np.array([e.x for e in grid.elements])
    assert np.allclose(xx, m["x"], rtol=1e-12, atol=0), tag + ": x"


def em_problem(s, window_ms=4.0, slice_thickness=1e-3, max_events=3000):
    """The inputs esvo_MVStereo hands its EventMatcher (esvo_MVStereo.cpp:579-608,1008-1040): the left / right events of the
    window before the observation stamp (at most EM_NUM_EVENT_MATCHING + 1 each), the left ones cut into slices of
    EM_Slice_Thickness with the pose at each slice's median stamp."""
    import indep_numpy as ind
    t_up = s["t_ts_ns"]; t_low = t_up - int(window_ms * 1e6)

    def window(e):
        lo = int(np.searchsorted(e["t"], t_low, side="left")); hi = int(np.searchsorted(e["t"], t_up, side="left")) - 1
        hi = min(hi, lo + max_events + 1)
        return {k: e[k][lo:hi].copy() for k in ("x", "y", "t", "p")}
    left, right = window(s["left"]), window(s["right"])
    counts, med = ind.event_slicing_for_em(left["t"], t_low, t_up, slice_thickness)
    poses = []
    for t in med:
        T = synth.pose_at(t * 1e-9)
        T[:3, 3] *= 1.0 if s["rig"] == "hkust" else 20.0     # synth.make_stream's scene scale
        poses.append(T.ravel())
    return left, right, counts, np.array(poses)


# ---- tracking (RegProblemSolverLM on one batch-sized block): one case table for the CPU pin and the device parity ----
# Defaults are the shipped hkust tracking yaml (Huber 50, kernelSize 5, 2 000 registration points, 10 iterations) with the
# rig's BATCH_SIZE; a case names only what it changes.  pose: exact | trans (prior off in translation, R_ = I) |
# rotx / roty / rotz (the reference frame 2-5 deg away from the current view, R_ != I) | far (the prior 2.5 deg and 6x
# the translation off).  img: scene | const (J == 0) | xonly (the TS varies along x only: dv == 0 exactly, so at
# R_ = I the t_y column of J is exactly zero; analytic only: the forward-difference t_y column is rounding noise).
# cloud: scene | off (every point off the image) | behind (half of the points mirrored behind the camera, projecting onto
# the same pixels) | line (see track_inputs).
TRACK_DEFAULT = dict(rig="hkust", an=True, B=None, reg=2000, n=6000, norm="huber50", k=5, it=10, pose="trans", img="scene",
                     cloud="scene")


def track_case_id(c):
    tag = [c["rig"], "B%d" % c["B"], c["norm"], "k%d" % c["k"], c["pose"]]
    for key, fmt in (("img", "%s"), ("cloud", "cloud-%s"), ("reg", "reg%d"), ("n", "n%d"), ("it", "it%d")):
        if c[key] != TRACK_DEFAULT[key]:
            tag.append(fmt % c[key])
    tag.append("an" if c["an"] else "num")
    return "-".join(tag)


def _tc(**kw):
    c = dict(TRACK_DEFAULT, **kw)
    if c["B"] is None:
        c["B"] = 500 if c["rig"] == "hkust" else 300
    c["id"] = track_case_id(c)
    return c


TRACK_CASES = [
    # the shipped configurations (the cases the suite ran before), analytic and numerical on every rig
    _tc(), _tc(an=False), _tc(rig="dsec"), _tc(rig="dsec", an=False), _tc(rig="upenn"), _tc(rig="upenn", an=False),
    # BATCH_SIZE: the minimum, one warp and a bit, below / at / above the block's 256 threads, up to TRK_MAXB
    _tc(B=6, img="xonly", cloud="line", it=20), _tc(B=32), _tc(B=33, norm="l2"), _tc(B=200, k=3), _tc(B=256, k=0), _tc(B=257, norm="huber5", k=3, pose="rotx"),
    _tc(B=1000, pose="roty"), _tc(B=1024, norm="l2", pose="rotz", an=False),
    # registration points: fewer than MAX_REGISTRATION_POINTS (n = 1 500), a cloud that is not a multiple of B, one batch,
    # more iterations than batches (the batch index wraps), 10 000 points (beyond the device's first allocation)
    _tc(n=1500, B=300, it=30), _tc(n=1234, reg=1234, B=1000), _tc(n=700, reg=700, B=700), _tc(reg=1100, B=257, it=30, norm="huber5"),
    _tc(n=12000, reg=10000, B=1024, it=2), _tc(rig="dsec", n=12000, reg=10000, B=1000, it=2, an=False),
    # norms, kernel sizes and MAX_ITERATION on the other rigs; rotation about every axis
    _tc(rig="dsec", norm="huber5", k=0, pose="rotx", it=30), _tc(rig="dsec", norm="l2", k=3, pose="rotz", it=1),
    _tc(rig="upenn", norm="huber5", k=3, pose="roty", it=2), _tc(rig="upenn", norm="l2", k=0, it=1, an=False),
    _tc(it=1, an=False), _tc(it=2, an=False, pose="rotx"), _tc(pose="exact"), _tc(pose="exact", an=False),
    # a large offset (2.5 deg and 6x the translation)
    _tc(pose="far"), _tc(pose="far", an=False, it=30), _tc(rig="dsec", pose="far", norm="huber5"),
    # constructed inputs
    _tc(img="const"), _tc(img="const", an=False), _tc(img="xonly", B=257, k=3), _tc(img="xonly", norm="l2", k=0, B=1024),
    _tc(cloud="off"), _tc(rig="upenn", cloud="off", an=False), _tc(cloud="behind"), _tc(cloud="behind", an=False, pose="rotz"),
]
assert len({c["id"] for c in TRACK_CASES}) == len(TRACK_CASES)
TRACK_CASES = {c["id"]: c for c in TRACK_CASES}

_TRACK_TS = {}


def _rot(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3)
    R[i, i] = c; R[j, j] = c; R[i, j] = -s; R[j, i] = s
    return R


def track_params(c, lib):
    p = configs.params_for(c["rig"], lib)
    p.trk_batch_size = c["B"]; p.trk_max_registration_points = c["reg"]; p.trk_max_iteration = c["it"]
    p.trk_kernel_size = c["k"]
    if c["norm"] == "l2":
        p.trk_lsnorm = capi.TRK_L2
    else:
        p.trk_lsnorm = capi.TRK_HUBER; p.trk_huber_threshold = float(c["norm"][5:])
    return p


def track_inputs(c, oracle_lib):
    """(left TS u8 H x W, float32 world cloud, T_world_ref, T_world_left prior) of one case; the cloud is a fresh copy."""
    rig = c["rig"]
    s = scenario(rig)
    l, r = configs.rig_calibs(rig)
    W, H = l.width, l.height
    if c["img"] == "scene":
        if rig not in _TRACK_TS:
            o = capi.Backend(oracle_lib, l, r, configs.params_for(rig, oracle_lib))
            _TRACK_TS[rig] = build_ts_pair(o, s)[0]
        tl = _TRACK_TS[rig]
    elif c["img"] == "const":
        tl = np.full((H, W), 93, np.uint8)
    else:
        x = np.arange(W)
        tl = np.repeat((128 + 100 * np.sin(x / 9.0) * np.cos(x / 31.0)).astype(np.uint8)[None, :], H, axis=0)
    scale = 1.0 if rig == "hkust" else 20.0
    Tw = np.asarray(s["T_world_left"], float).copy()
    if c["img"] == "xonly":
        Tw = np.eye(4)           # R_world_ref = R_world_left = I exactly: R_ = I, so J's t_y column is exactly 0
    rng = np.random.default_rng(11)
    pts = s["scene_points"]
    pc = (pts - Tw[:3, 3]) @ Tw[:3, :3]
    vis = np.nonzero(pc[:, 2] > 0.1)[0]
    sel = rng.choice(vis, size=min(c["n"], vis.size), replace=False)
    assert sel.size == c["n"], (c["id"], vis.size)
    cloud_cam = pc[sel]
    if c["cloud"] == "off":      # every point well outside the left image
        cloud_cam = cloud_cam.copy()
        cloud_cam[:, 0] = np.abs(cloud_cam[:, 0]) + 3.0 * cloud_cam[:, 2]
    elif c["cloud"] == "line":   # one horizontal line (Y within 1e-5 of Y0): at R_ = I, xonly makes the rotation-x / t_z and
        # rotation-z / t_x columns of J nearly parallel (exactly, were Y constant), so the QR's norm downdate re-computes
        Z = rng.uniform(0.8, 3.0, c["n"])
        cloud_cam = np.stack([rng.uniform(-0.8, 0.8, c["n"]) * Z, 0.3 * (1 + 1e-5 * rng.uniform(-1, 1, c["n"])), Z], axis=1)
    elif c["cloud"] == "behind":
        cloud_cam = cloud_cam.copy()
        cloud_cam[::2] *= -1.0
    cloud = (cloud_cam @ Tw[:3, :3].T + Tw[:3, 3]).astype(np.float32)
    T_ref, T_prior = Tw.copy(), Tw.copy()
    off = np.array([0.004, -0.003, 0.002]) * scale
    if c["pose"] == "trans":
        T_prior[:3, 3] += off
    elif c["pose"].startswith("rot"):
        axis = "xyz".index(c["pose"][3])
        T_ref[:3, :3] = Tw[:3, :3] @ _rot(axis, (2.0, 3.0, 5.0)[axis])
        T_ref[:3, 3] += np.array([0.01, 0.005, -0.008]) * scale
        T_prior[:3, 3] += off
    elif c["pose"] == "far":
        T_prior[:3, :3] = Tw[:3, :3] @ _rot(1, 2.5)
        T_prior[:3, 3] += 6 * off
    return tl, np.ascontiguousarray(cloud), T_ref, T_prior


def track_backend(c, lib, product_lib):
    """A context for case c on lib (oracle or product) that runs on the product's own rectification tables."""
    l, r = configs.rig_calibs(c["rig"])
    be = capi.Backend(lib, l, r, track_params(c, lib))
    if lib is not product_lib:
        for cam, calib in ((0, l), (1, r)):
            be.set_rectify_tables(cam, *capi.compute_rectify_tables(product_lib, calib))
    return be


TRACE_HEAD, TRACE_TRIAL = 22, 15


def track_trace(o):
    """esvo_oracle_track_trace of the last oracle solve: one dict per outer iteration, with its list of trials."""
    f = o.L.lib.esvo_oracle_track_trace
    f.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_size_t, C.POINTER(C.c_size_t)]
    f.restype = C.c_int
    n = C.c_size_t(0)
    f(o.ctx, None, 0, C.byref(n))
    buf = np.zeros(max(n.value, 1))
    assert f(o.ctx, buf.ctypes.data_as(C.POINTER(C.c_double)), buf.size, C.byref(n)) == 0
    out, i = [], 0
    while i < n.value:
        h = buf[i:i + TRACE_HEAD]; i += TRACE_HEAD
        it = dict(offset=int(h[0]), m=int(h[1]), status=int(h[2]), nfev=int(h[3]), rank=int(h[4]), nonzero_pivots=int(h[5]),
                  downdates=int(h[6]), fnorm=h[8], gnorm=h[9], R_=h[10:19].reshape(3, 3).copy(), t_=h[19:22].copy(), trials=[])
        for _ in range(int(h[7])):
            t = buf[i:i + TRACE_TRIAL]; i += TRACE_TRIAL
            it["trials"].append(dict(x=t[:6].copy(), fnorm1=t[6], actred=t[7], prered=t[8], ratio=t[9], par=t[10], delta=t[11],
                                     xnorm=t[12], accepted=bool(t[13]), lmpar_iter=int(t[14])))
        out.append(it)
    return out
