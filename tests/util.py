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


# ---- map side (fusion, clean, regularisation): one case table for the CPU pin (tests/test_map_pins.py) and the device
# parity (tests/test_gpu_map_parity.py).  Every case runs on the hkust rig (346 x 260); a case names only what it changes.
# norm: tdist | l2 | zncc (the map runs zncc through the Student-t path).  gen: the round-1 vector (map_round1).  pose:
# identity (J = 1, every propagated value exactly representable) | moved (a frame pose 3 deg / 2 cm away from the world
# and per-point observation poses a few degrees and centimetres from it).  r2: the second round, fused without a reset
# into the oracle's round-1 map (map_round2): thr (each decision of the case analysis placed on its threshold and one ulp
# either side) | regmap (after esvo_map_regularize: fusing into rho = -1 elements).
MAP_DEFAULT = dict(norm="tdist", radius=0, gen="lists", pose="identity", r2=None)
MAP_NORMS = {"tdist": capi.LSNORM_TDIST, "l2": capi.LSNORM_L2, "zncc": capi.LSNORM_ZNCC}


def _mc(**kw):
    c = dict(MAP_DEFAULT, **kw)
    tag = [c["norm"], "r%d" % c["radius"], c["gen"]]
    if c["pose"] != "identity":
        tag.append(c["pose"])
    if c["r2"]:
        tag.append("then-" + c["r2"])
    c["id"] = "-".join(tag)
    return c


MAP_CASES = [
    _mc(), _mc(radius=1), _mc(norm="l2"), _mc(norm="l2", radius=1), _mc(norm="zncc"),
    _mc(pose="moved"), _mc(norm="l2", pose="moved", radius=1), _mc(norm="zncc", pose="moved", radius=1),
    _mc(gen="edge"), _mc(gen="edge", radius=1), _mc(norm="l2", gen="edge"), _mc(norm="l2", gen="edge", radius=1),
    _mc(gen="guards"), _mc(gen="guards", radius=1),
    _mc(norm="l2", gen="l2floor"), _mc(norm="l2", gen="l2floor", radius=1),
    _mc(gen="bulk"), _mc(gen="bulk", radius=1, pose="moved"),
    _mc(gen="thr", r2="thr"), _mc(norm="l2", gen="thr", r2="thr"), _mc(gen="thr", r2="regmap"), _mc(norm="l2", gen="thr", r2="regmap"),
]
assert len({c["id"] for c in MAP_CASES}) == len(MAP_CASES)
MAP_CASES = {c["id"]: c for c in MAP_CASES}


def map_params(c, lib):
    p = configs.params_for("hkust", lib)
    p.lsnorm = MAP_NORMS[c["norm"]]
    p.fusion_radius = c["radius"]
    return p


def map_backends(c, oracle_lib, product_lib):
    return make_backends("hkust", oracle_lib, product_lib, tweak=lambda p: setattr(p, "lsnorm", MAP_NORMS[c["norm"]]))


def _nx(v, k):
    """v moved by k ulps."""
    for _ in range(abs(k)):
        v = float(np.nextafter(v, np.inf if k > 0 else -np.inf))
    return v


def depth_for(rho):
    """A depth z with 1.0 / z == rho exactly (None if no double within 64 ulps of 1 / rho has it)."""
    z0 = 1.0 / rho
    for k in range(65):
        for z in (_nx(z0, k), _nx(z0, -k)):
            if 1.0 / z == rho:
                return z
    return None


def map_point(Pl, u, v, rho, s2=0.0, nu=4.0, var=None, res=1.0, age=0, exact=True):
    """One DepthPoint (identity observation pose) that projects to pixel coordinates (u, v) of the left camera with inverse
    depth rho; exact=True picks its depth so that the propagation's 1 / z gives rho to the bit.  var defaults to
    nu / (nu - 2) * s2 (the Student-t variance; only the l2 propagation reads it)."""
    fx, cx, fy, cy = Pl[0][0], Pl[0][2], Pl[1][1], Pl[1][2]
    z = depth_for(rho) if exact else 1.0 / rho
    assert z is not None, rho
    q = np.zeros(1, capi.DEPTH_POINT_DTYPE)[0]
    q["p_cam"] = [(u - cx) / fx * z, (v - cy) / fy * z, z]
    q["row"], q["col"], q["x"], q["inv_depth"] = int(np.floor(v)), int(np.floor(u)), (u, v), rho
    q["scale2"], q["nu"] = s2, nu
    with np.errstate(all="ignore"):
        q["variance"] = var if var is not None else np.float64(nu) / (np.float64(nu) - 2) * np.float64(s2)
    q["residual"], q["age"] = res, age
    q["T_world_cam"] = np.eye(4).ravel()
    return q


def stack_points(qs):
    out = np.zeros(len(qs), capi.DEPTH_POINT_DTYPE)
    for i, q in enumerate(qs):
        out[i] = q
    return out


def _moved(pts, Pl, seed):
    """Re-express a vector built for identity poses under a frame pose T_wf 3 deg / 2 cm from the world: every point gets an
    observation pose T_wf * D (D: 1-4 deg, 0.5-2 cm) and the p_cam that puts it where it was in the frame."""
    rng = np.random.default_rng(seed)
    Tf = np.eye(4); Tf[:3, :3] = _rot(1, 3.0) @ _rot(0, -1.5); Tf[:3, 3] = [0.02, -0.01, 0.015]
    out = pts.copy()
    for q in out:
        D = np.eye(4); D[:3, :3] = _rot(int(rng.integers(0, 3)), rng.uniform(1, 4)); D[:3, 3] = rng.uniform(-0.02, 0.02, 3)
        Twc = Tf @ D
        p_f = np.append(q["p_cam"], 1.0)
        q["p_cam"] = (np.linalg.inv(D) @ p_f)[:3]
        q["T_world_cam"] = Twc.ravel()
    return out, Tf


def _edge_points(Pl, W, H):
    """Projections whose splat leaves the image, x just below 0, a NaN re-projection, points behind the camera that project
    into the image (elements with rho < -1e-6) and, later in the vector, compatible contributions into them (the "new point"
    branch), each with a second contribution so that the fusion runs there too."""
    qs = []
    for (u, v) in ((W - 1e-9, 100.5), (W - 0.5, 37.25), (170.5, H - 1e-9), (60.3, H - 0.5), (W - 1e-7, H - 1e-7), (0.0, 0.0),
                   (0.25, 120.5), (200.5, 0.0)):
        qs += [map_point(Pl, u, v, 0.8, s2=2e-4, nu=2.1897, res=5.0), map_point(Pl, u, v, 0.81, s2=1e-4, nu=2.1897, res=4.0)]
    qs.append(map_point(Pl, -1e-9, 50.5, 0.7, s2=1e-4, exact=False))        # x just below 0: outside
    qs.append(map_point(Pl, 50.5, -1e-9, 0.7, s2=1e-4, exact=False))
    nan = map_point(Pl, 80.5, 80.5, 0.7, s2=1e-4); nan["p_cam"] = 0.0       # h = (0, 0, 0): 0 / 0 re-projection
    qs.append(nan)
    for i, (u, v) in enumerate(((120.5, 60.5), (240.5, 180.5), (30.5, 200.5), (W - 0.5, H - 0.5))):
        qs.append(map_point(Pl, u, v, -0.5 - 0.25 * i, s2=1e-4, res=3.0))      # behind the camera, lands in the image
        qs.append(map_point(Pl, u, v, 0.6, s2=2.0, nu=2.1897, res=9.0))        # 2 sigma > |0.6 - rho|: the "new point" branch
        qs.append(map_point(Pl, u, v, 0.61, s2=1e-3, nu=2.1897, res=2.0))      # then an ordinary update of the new point
    for i, rho in enumerate((_nx(-1e-6, -1), -1e-6, _nx(-1e-6, 1))):              # the validity threshold and its neighbours
        qs.append(map_point(Pl, 280.5 + 20 * i, 200.5, rho, s2=1e-4, res=3.0))
    qs.append(map_point(Pl, 140.5, 140.5, -1.0, s2=1e-4, res=3.0))              # rho = -1 exactly, then far contributions
    qs.append(map_point(Pl, 140.5, 140.5, 0.7, s2=1e-6, res=1.0))               # not compatible: case 2.2 against rho = -1
    return stack_points(qs)


def _guard_points(Pl):
    """Pairs (map element, then one update) on separate pixels that take each arm of the fast path's guards: S below 1e-200
    and above 1e200, nu_u = 2 exactly (var = +inf), just above 2, below 2 (a negative variance: NaN sigma and a NaN
    compatibility test), >= 1e15, denormal scale, and updates whose variance leaves (1e-200, 1e200) (sqrt vs sqrt_nr)."""
    pairs = [
        ((0.5, 4e-201, 3.0), (0.5000001, 5e-201, 3.0)),      # S < 1e-200
        ((0.5, 1e-200, 3.0), (0.5000001, 2e-200, 3.0)),      # S just above 1e-200, variance below 1e-200 after the update
        ((0.5, 6e199, 3.0), (0.5000001, 6e199, 3.0)),        # S > 1e200
        ((0.5, 4e199, 3.0), (0.5, 4e199, 3.0)),              # S < 1e200
        ((1e101, 4e199, 2.05), (1.09e101, 4e199, 2.05)),     # fast path, variance above 1e200 after the update
        ((0.5, 1e-3, 2.0), (0.52, 1e-3, 2.0)),               # nu_u = 2: var = +inf, sigma = inf
        ((0.5, 1e-3, 2.0 + 2e-15), (0.52, 1e-3, 5.0)),       # just above 2
        ((0.5, 1e-3, 4.0), (0.52, 1e-3, 0.5)),               # nu_u = 0.5: after the update nu = 1.5 -> var < 0 -> NaN sigma
        ((0.5, 1e-3, 4.0), (0.51, 1e-3, 1.5)),               # the propagated point's own var < 0 (NaN 2 sigma)
        ((0.5, 1e-3, 1e15), (0.51, 1e-3, 2e15)),             # nu_u >= 1e15
        ((0.5, 1e-3, 3e14), (0.51, 1e-3, 4e14)),             # just below
        ((0.5, 1e-310, 3.0), (0.5, 1e-3, 3.0)),              # denormal scale of the map point (S normal)
        ((0.5, 1e-3, 3.0), (0.5000001, 3e-312, 3.0)),        # denormal scale of the propagated point
        ((0.5, 1e-310, 3.0), (0.5, 1e-309, 3.0)),            # both denormal (S < 1e-200)
        ((0.5, 2e-190, 3.0), (0.5000001, 3e-190, 3.0)),      # s2 * s2 underflows to a denormal in the numerator
        ((1e-310, 1e-3, 3.0), (2e-310, 1e-3, 3.0)),          # denormal inverse depths
    ]
    qs, pts_next = [], []
    for i, ((r0, s0, n0), (r1, s1, n1)) in enumerate(pairs):
        u, v = 20.5 + 25 * (i % 12), 20.5 + 40 * (i // 12)
        qs.append(map_point(Pl, u, v, r0, s2=s0, nu=n0, res=2.0, exact=False))
        pts_next.append(map_point(Pl, u, v, r1, s2=s1, nu=n1, res=1.0, exact=False))
        pts_next.append(map_point(Pl, u, v, r1, s2=s1 * 1.5, nu=n1 + 1.0, res=0.5, exact=False))   # one more update on top
    return stack_points(qs + pts_next)


def _l2floor_points(Pl):
    """l2: variances below 1e-6 on create (the propagation's floor), fuse (the update's floor) and replace."""
    qs = []
    for i, (v0, v1, r1) in enumerate(((1e-7, 2e-7, 0.5), (1.5e-6, 1.5e-6, 0.5), (1e-6, 1e-6, 0.5), (4e-6, 1e-8, 0.5 + 0.01),
                                      (3e-6, 5e-7, 0.6), (2e-6, 1e-12, 0.4))):
        u, v = 30.5 + 40 * i, 60.5
        qs.append(map_point(Pl, u, v, 0.5, var=v0, res=3.0))
        qs.append(map_point(Pl, u, v, r1, var=v1, res=1.0))
    return stack_points(qs)


def _bulk_points(Pl, seed=3):
    """24 contributions on each of 200 pixels, all in one inverse-depth cluster: thousands of Student-t updates through the
    fast path (rcp_nr / div_nr / sqrt_nr), compared bit for bit."""
    rng = np.random.default_rng(seed)
    qs = []
    for i in range(200):
        row, col = 12 + 24 * (i // 25), 12 + 13 * (i % 25)
        for _ in range(24):
            rho = 0.7 * (1 + 0.01 * rng.standard_normal())
            s2 = (10 ** rng.uniform(-2.5, -1.0)) ** 2
            qs.append(map_point(Pl, col + rng.uniform(0.1, 0.9), row + rng.uniform(0.1, 0.9), rho, s2=s2, nu=2.1897,
                                var=s2 * 2.1897 / 0.1897, res=rng.uniform(1, 50), age=int(rng.integers(0, 3)), exact=False))
    pts = stack_points(qs)
    return pts[rng.permutation(pts.size)]


THR_RHO = 0.5625            # 9/16; with nu = 4 the Student-t variance 2 * s2 and 2 sigma are exact powers of two
THR_S2 = 2.0 ** -15         # var = 2^-14, 2 sigma = 2^-6
THR_TINY_S2 = 2.0 ** -41    # 2 sigma = 2^-19


def _thr_base(Pl, norm):
    """Round 1 of the threshold cases: one element block per target (a 2 x 2 splat of one point), columns of 11 px."""
    qs = []
    for i, kind in enumerate(THR_KINDS):
        u, v = 15.5 + 11 * (i % 30), 30.5 + 30 * (i // 30)
        s2 = THR_TINY_S2 if kind[0] == "prop2s" else THR_S2
        qs.append(map_point(Pl, u, v, THR_RHO, s2=s2, nu=4.0, var=2 * s2, res=2.0, age=1))
    return stack_points(qs)


# (decision, offset in ulps of the placed quantity): the round-2 contribution of each target pixel
THR_KINDS = [(k, o) for k in ("map2s", "prop2s", "occl", "chi") for o in (-1, 0, 1)] + \
            [("tie", o) for o in ("eq", "var", "res", "both")]


def _thr_round2(m, Pl, norm):
    """Round 2 of the threshold cases, from the round-1 map m (the oracle's): per target, one contribution placed on the
    threshold of one decision (or one ulp off it), in f64 computed in the reference's order."""
    qs = []
    cell = {(int(e["row"]), int(e["col"])): e for e in m}
    for i, (kind, off) in enumerate(THR_KINDS):
        u, v = 15.5 + 11 * (i % 30), 30.5 + 30 * (i // 30)
        e = cell[(int(np.floor(v)), int(np.floor(u)))]
        rho0, var0 = float(e["inv_depth"]), float(e["variance"])
        sdm = 2 * np.sqrt(var0)
        if kind == "map2s":       # |prho - rho| == 2 sigma of the map point (+-1 ulp); the propagated point's own 2 sigma tiny
            rho = _nx(rho0 + sdm, off)
            assert off != 0 or abs(rho - rho0) == sdm
            qs.append(map_point(Pl, u, v, rho, s2=THR_TINY_S2, var=2 * THR_TINY_S2, res=3.0))
        elif kind == "prop2s":    # |prho - rho| == 2 sigma of the propagated point; the map point's tiny
            sd2 = 2 * np.sqrt(2 * THR_S2)
            rho = _nx(rho0 - sd2, -off)
            assert off != 0 or abs(rho - rho0) == sd2
            qs.append(map_point(Pl, u, v, rho, s2=THR_S2, var=2 * THR_S2, res=3.0))
        elif kind == "occl":      # rho - 2 sigma == prho (+-1 ulp): not compatible at and below, compatible above
            rho = _nx(rho0 - sdm, off)
            assert off != 0 or rho0 - sdm == rho
            qs.append(map_point(Pl, u, v, rho, s2=THR_S2, var=var0 if norm == "l2" else 2 * THR_S2, res=1.0))
        elif kind == "chi":       # d2 / pvar + d2 / var on either side of 5.99 (pvar = var), searched over the depths
            def chi(z):
                d2 = (1.0 / z - rho0) * (1.0 / z - rho0)
                return d2 / var0 + d2 / var0
            z = 1.0 / (rho0 + np.sqrt(5.99 * var0 / 2))      # a larger depth: a smaller prho - rho0 and chi
            while chi(z) < 5.99:
                z = _nx(z, -1)
            while chi(_nx(z, 1)) >= 5.99:
                z = _nx(z, 1)
            # z: the last depth with chi >= 5.99; off -1 -> the next one (chi < 5.99), +1 -> the one before (chi above)
            rho = 1.0 / _nx(z, -off)
            qs.append(map_point(Pl, u, v, rho, s2=THR_S2, var=var0, res=3.0))
        else:                     # replace test on ties: pvar == var and / or pres == res (not compatible, not occluded)
            rho = rho0 + 10 * sdm
            s2 = THR_S2 if off in ("eq", "res") else _nx(THR_S2, -1)
            res = float(e["residual"]) if off in ("eq", "var") else _nx(float(e["residual"]), -1)
            var = 2 * s2
            qs.append(map_point(Pl, u, v, rho, s2=s2, var=var, res=res))
    return stack_points(qs)


def _reg_round2(m, Pl, norm):
    """After esvo_map_regularize rejected the isolated round-1 elements (rho = -1): contributions whose 2 sigma reaches -1
    (the "new point" branch) and narrow ones (case 2.2 against rho = -1)."""
    qs = []
    for k, e in enumerate(m):
        if k % 4:
            continue
        u, v = float(e["col"]) + 0.5, float(e["row"]) + 0.5
        if (k // 4) % 2 == 0:
            qs.append(map_point(Pl, u, v, 0.6, s2=1.0, nu=4.0, var=4.0, res=1.0))
        else:
            qs.append(map_point(Pl, u, v, 0.6, s2=1e-4, nu=4.0, var=1e-4, res=1.0))
    return stack_points(qs)


def map_round1(c, Pl, W=346, H=260):
    """(points, T_world_frame) of the case's first round (fused with reset_map = 1)."""
    gen = c["gen"]
    if gen == "lists":
        pts, _ = fold_vector(Pl, lengths=(1, 2, 3, 33, 65, 70, 193, 200), seed=7)
    elif gen == "edge":
        pts = _edge_points(Pl, W, H)
    elif gen == "guards":
        pts = _guard_points(Pl)
    elif gen == "l2floor":
        pts = _l2floor_points(Pl)
    elif gen == "bulk":
        pts = _bulk_points(Pl)
    else:
        pts = _thr_base(Pl, c["norm"])
    if c["norm"] == "l2" and gen in ("lists", "bulk"):
        pts["variance"] = pts["scale2"] * 2.0
    T = np.eye(4)
    if c["pose"] == "moved":
        pts, T = _moved(pts, Pl, seed=5)
    return pts, T


def map_round2(c, m, Pl):
    """The second-round points of case c (fused with reset_map = 0), built from the round-1 map m; None for one-round cases."""
    if c["r2"] == "thr":
        return _thr_round2(m, Pl, c["norm"])
    if c["r2"] == "regmap":
        return _reg_round2(m, Pl, c["norm"])
    return None


def map_vec(pts):
    """A point vector as the dicts tests/indep_fusion.py reads."""
    return [dict(p_cam=q["p_cam"], s2=float(q["scale2"]), nu=float(q["nu"]), var=float(q["variance"]), res=float(q["residual"]),
                 age=int(q["age"]), T_world_cam=q["T_world_cam"]) for q in pts]


MAP_F64 = ("inv_depth", "scale2", "nu", "variance", "residual", "x")


def bits_equal(a, b):
    """Element-wise: the same f64 bits, or both NaN (x86 and the GPU produce different default NaN payloads)."""
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def maps_bit_identical(mo, mg, tag, p_cam_rtol=1e-12):
    """Two downloaded maps: size, element order, rows / cols, ages exact; every f64 field but p_cam bit-identical; p_cam
    within p_cam_rtol (closed-form cam2World on the device, DESIGN.md deviation 3)."""
    assert mo.size == mg.size, (tag, mo.size, mg.size)
    assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"]), tag + ": element order"
    assert np.array_equal(mo["age"], mg["age"]), tag + ": ages"
    for f in MAP_F64:
        eq = bits_equal(mo[f], mg[f])
        assert eq.all(), (tag, f, int((~eq).sum()), np.nonzero(~eq.reshape(len(mo), -1).all(axis=1))[0][:5],
                          mo[f][~eq][:3], mg[f][~eq][:3])
    pc_o, pc_g = mo["p_cam"], mg["p_cam"]
    fin = np.isfinite(pc_o)
    assert np.array_equal(fin, np.isfinite(pc_g)), tag + ": p_cam finiteness"
    assert np.allclose(pc_g[fin], pc_o[fin], rtol=p_cam_rtol, atol=1e-300), (tag, "p_cam", np.abs(pc_g[fin] - pc_o[fin]).max())


# ---- depth LM, Student-t scale iteration: one hand-built case table for the CPU restatement (tests/test_depth_irls_pins.py)
# and the device parity (tests/test_gpu_depth_irls.py).  Every case runs on the hkust rig with T_world_left =
# T_world_virtual = identity.  The right time surface is the left one shifted by D pixels; the seed sits at (x + 0.5, y) with
# y a whole row, so the lower tap row has weight exactly 0 and every patch row is independent; its inverse depth puts the
# right patch delta pixels off, so pixel k's residual is delta * g_k for the integer horizontal gradient g_k the case draws
# (the image values stay within 0..63, so the taps of zero gradients cancel exactly).  nz and min |r| are thus chosen, and
# nu places c = (nu+1) nz / N against 0.95 (eps = 1 - c / 0.95).  big = (E, k): the right surface is raised by E under the
# first k pixels, residuals of about -E among the small ones.
DEPTH_DEFAULT = dict(patch=(15, 7), nz=28, g=1, delta=1.5e-6, nu=2.182, scale=17.277, eps=None, ulp=0, big=None, D=10, x=100,
                     y=130, edge=False)


def _dc(name, **kw):
    c = dict(DEPTH_DEFAULT, **kw)
    c["id"] = name
    N = c["patch"][0] * c["patch"][1]
    if c.get("below_095"):                               # the largest nu with (nu+1) nz < 0.95 N: inside the 1e-9 margin
        nz, T = c["below_095"], 0.95 * float(N)
        nu = T / nz - 1.0
        while (nu + 1) * float(nz) >= T:
            nu = float(np.nextafter(nu, -np.inf))
        c["nu"] = nu
    elif c["eps"] is not None or c["ulp"]:               # nu with (nu+1) nz = 0.95 N (1 - eps), or on the 1e-9 margin +- ulps
        nz = c["nz"]
        if c["eps"] is not None:
            c["nu"] = 0.95 * N * (1.0 - c["eps"]) / nz - 1.0
        else:
            T = 0.95 * float(N) * (1.0 - 1e-9)
            nu = T / nz - 1.0
            while (nu + 1) * float(nz) < T:
                nu = float(np.nextafter(nu, np.inf))
            while (nu + 1) * float(nz) >= T:
                nu = float(np.nextafter(nu, -np.inf))
            # nu is now the largest value the guard's "<" accepts; ulp = +1 is the first it declines
            c["nu"] = nu if c["ulp"] < 0 else float(np.nextafter(nu, np.inf))
            c["ulp_at"] = c["ulp"]
    return c


DEPTH_CASES = [
    # the shipped shape and both shipped nu (c = 0.85): the shortcut's common path, and non-degenerate controls
    _dc("15x7-shipped-dsec"), _dc("15x7-shipped-hkust", nu=2.1897, scale=16.6397),
    _dc("15x7-nondeg-1pass", nz=105, big=(17, 105), delta=1e-3), _dc("15x7-nondeg-2pass", nz=105, big=(16, 105), delta=1e-3),
    _dc("15x7-nondeg-4pass", nz=105, big=(2, 105), delta=1e-3), _dc("15x7-c-above-0.95", nz=32, delta=1e-3),
    _dc("15x7-mixed-big-tiny", nz=40, big=(40, 10), delta=1e-6),
    # the band of the issue: 67 x 1 and 1 x 67 with 20 unit gradients at the shipped dsec nu (eps = 1.6e-4)
    _dc("67x1-band-1.5e-6", patch=(67, 1), nz=20), _dc("67x1-reset-3e-6", patch=(67, 1), nz=20, delta=3e-6),
    _dc("67x1-rmin-0.99e-6", patch=(67, 1), nz=20, delta=0.99e-6), _dc("67x1-rmin-1.01e-6", patch=(67, 1), nz=20, delta=1.01e-6),
    _dc("1x67-band-1.5e-6", patch=(1, 67), nz=20, x=30, y=100), _dc("67x1-rmin-1e-4", patch=(67, 1), nz=20, delta=1e-4),
    # a stall whose last subnormal step shrinks the scale by exactly 1/20: the division arm's "> 0.05" ends the loop there
    _dc("67x1-stall-at-exact-5pct", patch=(67, 1), nz=20, delta=1.001500500166722e-06),
    # eps placed at 1e-8 .. 1e-2 at N = 105, nz = 32, r_min = 3e-6; the 1e-9 margin itself and one ulp above it
    *[_dc(f"15x7-eps{e:g}", nz=32, delta=3e-6, eps=e) for e in (1e-8, 1e-6, 1e-4, 1e-3, 1e-2)],
    _dc("15x7-eps1e-6-rmin1.2e-6", nz=32, delta=1.2e-6, eps=1e-6), _dc("15x7-eps1e-6-rmin1e-5", nz=32, delta=1e-5, eps=1e-6),
    _dc("15x7-eps1e-8-rmin1e-4", nz=32, delta=1e-4, eps=1e-8),
    _dc("15x7-margin-accepted", nz=32, delta=3e-6, ulp=-1), _dc("15x7-margin-declined", nz=32, delta=3e-6, ulp=1),
    # c one ulp below 0.95, inside the 1e-9 margin, with residuals of about -10 on 33 pixels: gap * min r^2 passes the reset bound,
    # but the literal loop ends through a 5 % test decided at rounding level near a scale of 1e-15 (no reset)
    _dc("15x7-inside-margin-big", nz=0, big=(10, 32), below_095=33),
    # residuals below the old guard's 1e-6: the device's literal loops
    _dc("15x7-rmin-1e-7", delta=1e-7), _dc("15x7-rmin-1e-8", delta=1e-8),
    # lm2_kernel at m < 16 and lm_kernel<8, true> at 113, 121 and 127 pixels
    _dc("1x1-nondeg", patch=(1, 1), nz=1, delta=1e-3), _dc("3x3-deg", patch=(3, 3), nz=2, delta=1e-5),
    _dc("3x3-band", patch=(3, 3), nz=2, delta=3e-6, eps=1e-6),
    _dc("113x1-band", patch=(113, 1), nz=32, delta=3e-6, eps=1e-6, x=110), _dc("113x1-shipped-nu", patch=(113, 1), nz=30, x=110),
    _dc("11x11-band", patch=(11, 11), nz=36, delta=3e-6, eps=1e-6), _dc("11x11-shipped-nu", patch=(11, 11), nz=30),
    _dc("127x1-band", patch=(127, 1), nz=36, delta=3e-6, eps=1e-6, x=110), _dc("127x1-eps1e-3", patch=(127, 1), nz=36, delta=3e-6, eps=1e-3, x=110),
    # the right patch against the image's left edge: the warp holds at x0 and fails at x0 + h
    _dc("15x7-warp-fails-at-x0+h", edge=True),
]
assert len({c["id"] for c in DEPTH_CASES}) == len(DEPTH_CASES)
DEPTH_CASES = {c["id"]: c for c in DEPTH_CASES}


def depth_params(c, lib, max_iteration=10):
    p = configs.params_for("hkust", lib)
    p.lsnorm = capi.LSNORM_TDIST
    p.patch_size_x, p.patch_size_y = c["patch"]
    p.td_nu, p.td_scale = c["nu"], c["scale"]
    p.max_iteration = max_iteration
    return p


@functools.lru_cache(maxsize=None)
def depth_inputs(cid):
    """(tl, tr, seed, x_seed, y_seed) of DEPTH_CASES[cid]: the time surfaces, one seed (SEED_DTYPE) and its pixel position."""
    import indep_depth as idp
    c = DEPTH_CASES[cid]
    A = configs.rig_arrays("hkust")
    W, H = A["width"], A["height"]
    Pl, Pr = A["left"]["P"], A["right"]["P"]
    wx, wy = c["patch"]
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    N, D = wx * wy, c["D"]
    x, y = c["x"], c["y"]
    fb = -Pr[0][3]
    if c["edge"]:
        x = hx + D                                         # right patch centre 5e-8 px right of hx: x0 + h moves it 1.6e-7 px left
        rho0 = (x + 0.5 - hx - 5e-8) / fb
    else:
        rho0 = (D + c["delta"]) / fb
    # the inverse depth nearest rho0 at which the kernels' closed-form cam2World and the reference's literal one agree to the bit
    cand = [rho0]
    for k in range(1, 200):
        cand += [_nx(rho0, k), _nx(rho0, -k)]
    rho = None
    for r in cand:
        pd, pl = idp.cam2world_device(Pl, x + 0.5, float(y), r), idp.cam2world_literal(Pl, x + 0.5, float(y), r)
        a1, a2 = idp.project(Pl, pd), idp.project(Pr, pd)
        if a1 == idp.project(Pl, pl) and a2 == idp.project(Pr, pl) and a1 == (x + 0.5, float(y)):
            rho = r
            break
    assert rho is not None, cid
    # per-pixel gradients: nz pixels spread evenly over the patch (row-major), sign alternating along each row
    g = np.zeros(N, np.int64)
    g[np.round(np.linspace(0, N - 1, c["nz"])).astype(int) if c["nz"] else []] = c["g"]
    g = g.reshape(wy, wx)
    L = np.full((H, W), 32, np.int64)
    ulx, uly = x - hx, y - hy
    for py in range(wy):
        row = uly + py
        for px in range(wx):
            s = 1 if px % 2 == 0 else -1
            L[row, ulx + px + 1] = L[row, ulx + px] + s * g[py, px]
        L[row, ulx + wx + 1:] = L[row, ulx + wx]
    assert L.min() >= 0 and L.max() <= 63
    R = np.full_like(L, 32)
    R[:, :W - D] = L[:, D:]
    if c["big"]:
        E, k = c["big"]
        for q in range(k):
            py, px = divmod(q, wx)
            R[uly + py, ulx - D + px:ulx - D + px + 2] = L[uly + py, ulx + px:ulx + px + 2] + E
    seed = np.zeros(1, capi.SEED_DTYPE)
    seed["x_left"] = seed["x_left_raw"] = (x + 0.5, float(y))
    seed["T_world_virtual"] = np.eye(4).ravel()
    seed["inv_depth"] = rho
    return L.astype(np.uint8), R.astype(np.uint8), seed, x + 0.5, float(y)


# ---- time-surface cases: push / build scripts that reach every branch of ts_push and ts_run_build (esvo_b200/csrc/ts.cu) ----
# A case is (size, parameter tweak, script).  The script is a list of ops run on the oracle and on the product alike:
#   ("push", how, ev)          how: host | nopol | dev | devnopol | packet (four adjacent host arrays) | packetnopol (three, pol = NULL)
#   ("build", T)               index grid and image of both sides must be equal
#   ("refused", T, code)       the product's esvo_ts_build must return `code`
#   ("push_refused", ev, code) the product's push must return `code`; nothing is pushed on either side
#   ("sync",) ("reset",)       esvo_sync (product) / esvo_ts_reset (both)
#   ("unordered", on)          esvo_ts_set_unordered_input (product; the oracle always handles any order)
#   ("unordered_refused",)     switching it on must return ESVO_ERR_UNSUPPORTED
#   ("fresh", ev, T)           a new product context fed ev must build at T what this one built last
TS_UNSUPPORTED, TS_CAPACITY = -6, -4
TS_LOG_CAP = 1 << 22                       # resident events per camera (ts_alloc); a fold keeps TS_LOG_CAP / 4
TS_EPOCH = 1_600_000_000_000_000_000       # a UNIX-epoch stamp in ns: 2.4e-7 s between neighbouring doubles
TS_SIZES = {"hkust": (346, 260), "dsec": (640, 480), "small": (120, 96), "odd": (223, 165)}


def ts_rig(size):
    """Name under configs.RIGS: the shipped rigs, the small rig of the golden vectors, and hkust scaled to 223 x 165 (W % 32 = 31,
    H % 8 = 5: partial tiles on both axes of the 32 x 8 raster kernels)."""
    if size == "small" and "golden_small" not in configs.RIGS:
        import ast
        import os
        z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "small_rig_frame.npz"), allow_pickle=False)
        configs.RIGS["golden_small"] = ast.literal_eval(bytes(z["rig_json"]).decode())
    if size == "odd" and "hkust_odd" not in configs.RIGS:
        W, H = TS_SIZES["odd"]
        h = configs.RIGS["hkust"]
        sx, sy = W / h["width"], H / h["height"]
        def scaled(c):
            K = np.array(c["K"], float).reshape(3, 3); P = np.array(c["P"], float).reshape(3, 4)
            K[0] *= sx; K[1] *= sy; P[0] *= sx; P[1] *= sy
            return dict(K=K.ravel().tolist(), D=c["D"], R=c["R"], P=P.ravel().tolist())
        configs.RIGS["hkust_odd"] = dict(width=W, height=H, model="plumb_bob", left=scaled(h["left"]), right=scaled(h["right"]))
    return {"small": "golden_small", "odd": "hkust_odd"}.get(size, size)


def ts_ev(x, y, t, p=None):
    x = np.asarray(x, np.uint16)
    return dict(x=x, y=np.asarray(y, np.uint16), t=np.asarray(t, np.int64), p=np.ones(x.size, np.uint8) if p is None else np.asarray(p, np.uint8))


def ts_cut(ev, a, b):
    return {k: v[a:b] for k, v in ev.items()}


def ts_cat(*evs):
    return {k: np.concatenate([e[k] for e in evs]) for k in ("x", "y", "t", "p")}


def ts_random_stream(W, H, n, seed, t0=1_000_000_000, dt=2000):
    """Time-ordered (equal stamps allowed); half of the events fall on a 24 x 16 patch, so its pixels hold more than any queue."""
    rng = np.random.default_rng(seed)
    x = rng.integers(0, W, n); y = rng.integers(0, H, n)
    hot = rng.random(n) < 0.5
    x[hot] = W // 3 + rng.integers(0, 24, hot.sum()); y[hot] = H // 3 + rng.integers(0, 16, hot.sum())
    return ts_ev(x, y, t0 + np.cumsum(rng.integers(0, 2 * dt, n)), rng.integers(0, 2, n))


def ts_jitter(ev, seed, frac=0.08, max_ns=2_000_000):
    """A fraction of the events arrives with a stamp up to max_ns in the past."""
    rng = np.random.default_rng(seed)
    t = ev["t"].copy()
    late = rng.random(t.size) < frac
    late[0] = False
    t[late] -= rng.integers(1_000, max_ns, late.sum())
    return dict(ev, t=t)


def _pushes(ev, sizes, how="host"):
    ops, a = [], 0
    for k, n in enumerate(sizes):
        b = ev["t"].size if n is None else a + n
        ops.append(("push", how[k % len(how)] if isinstance(how, (list, tuple)) else how, ts_cut(ev, a, b)))
        a = b
    assert a == ev["t"].size
    return ops


def _builds(ev, extra=()):
    t = np.sort(ev["t"])
    return [("build", int(t[-1]) + 1), ("build", int(t[t.size // 2])), ("build", int(t[t.size // 5]))] + [("build", int(T)) for T in extra]


def _s_plain(W, H, how="host", n=30000, seed=11):
    ev = ts_random_stream(W, H, n, seed)
    return _pushes(ev, [n // 3, 7, None], how) + _builds(ev)


TS_QLEN_PIX = ((3, 2), (5, 2), (7, 2))     # hold qlen - 1, qlen, qlen + 1 events that are not older than TS_QLEN_T
TS_QLEN_T = 1_030_000_000


def _s_qlen(W, H, q):
    bg = ts_random_stream(W, H, 6000, 21)
    keep = ~((bg["y"] == 2) & (bg["x"] < 10))
    bg = {k: v[keep] for k, v in bg.items()}
    xs, ys, tt = [], [], []
    for k, (px, py) in enumerate(TS_QLEN_PIX):
        n_new = q - 1 + k
        xs += [px] * (2 + n_new); ys += [py] * (2 + n_new)
        tt += [TS_QLEN_T - 5000 - k, TS_QLEN_T - 1] + [TS_QLEN_T + 700 * j for j in range(n_new)]   # the first new one AT T: not "< T"
    sp = ts_ev(xs, ys, tt, [(i * 7) % 3 != 0 for i in range(len(xs))])
    ev = ts_cat(bg, sp)
    o = np.argsort(ev["t"], kind="stable")
    ev = {k: v[o] for k, v in ev.items()}
    return _pushes(ev, [ev["t"].size // 2, None]) + [("build", TS_QLEN_T), ("build", TS_QLEN_T + 1), ("build", int(ev["t"][-1]) + 1)]


def _s_t_edges(W, H):
    ev = ts_random_stream(W, H, 20000, 31)
    ev["t"][9000:9005] = ev["t"][9004]                                     # five events share one stamp
    ev["t"][:3] = ev["t"][0]; ev["t"][-3:] = ev["t"][-1]                   # so do the oldest and the newest three
    t = ev["t"]
    return [("build", 1_500_000_000)] + _pushes(ev, [12000, None]) + \
           [("build", int(T)) for T in (t[-1], t[-1] + 1, t[0], t[0] + 1, t[9004], t[9004] + 1)] + [("reset",), ("build", int(t[-1]))]


def _s_stamp0_offimage_epoch(W, H):
    head = ts_ev([5, 6, W, 3, 65535, 6, 9, W - 1], [5, 5, 3, H, 65535, 5, H - 1, 65535], [0, 0, 10, 20, 30, 40, 50, 60], [1, 0, 1, 1, 0, 0, 1, 1])
    body = ts_random_stream(W, H, 8000, 41, t0=TS_EPOCH, dt=40)            # neighbouring stamps fall on the same double
    body["x"][1000::997] = W; body["y"][1500::997] = H
    ev = ts_cat(head, body)
    t = body["t"]
    return _pushes(ev, [5, 2000, None]) + [("build", int(T)) for T in (1, 41, 61, t[0], t[4000], t[4000] + 1, t[-1] + 1)]


def _s_dev(W, H, kind):
    ev = ts_random_stream(W, H, 30000, 51)
    n, t = 30000, ev["t"]
    if kind in ("dev", "devnopol"):
        return _pushes(ev, [n // 2, None], kind) + _builds(ev)
    if kind == "dev-then-host":
        return _pushes(ev, [n // 2, None], ["dev", "host"]) + _builds(ev, [t[-1]])
    a, b = ts_cut(ev, 0, 10000), ts_cut(ev, 10000, 20000)                  # dev-drain-then-build
    return [("push", "dev", a), ("sync",), ("build", int(t[9999]) + 1), ("build", int(t[9999])), ("build", int(t[5000])),
            ("push", "host", b), ("build", int(t[19999]) + 1), ("build", int(t[19999])),
            ("push", "dev", ts_cut(ev, 20000, n)), ("build", int(t[-1]) + 1), ("build", int(t[15000]))]


def _s_packet(W, H):
    ev = ts_random_stream(W, H, 4095 + 4096 + 4096 + 5000, 61)
    return _pushes(ev, [4095, 4096, 4096, None], ["packet", "packet", "packetnopol", "packet"]) + _builds(ev)


def _s_unord(W, H, kind):
    on = [("unordered", 1)]
    if kind == "ties":            # 50 distinct stamps in random arrival order: ties with the running maximum, the later arrival wins
        rng = np.random.default_rng(71)
        n = 3000
        ev = ts_ev(rng.integers(0, W, n), rng.integers(0, H, n), 1_000_000_000 + 1000 * rng.integers(0, 50, n), rng.integers(0, 2, n))
        return on + _pushes(ev, [1500, None]) + [("build", 1_000_050_000), ("build", 1_000_049_000), ("build", 1_000_025_000)]
    if kind == "carry-wins-blocks":   # three whole scan blocks older than the event carried from the first push
        first = ts_ev([10, 11, 12], [20, 20, 20], [1_000_000_000, 1_900_000_000, 1_000_000_500], [1, 0, 1])
        older = ts_random_stream(W, H, 3072, 72, t0=1_100_000_000)
        mixed = ts_random_stream(W, H, 2500, 73, t0=1_899_000_000, dt=1000)   # crosses the carried stamp half-way
        assert older["t"].max() < 1_900_000_000 < mixed["t"].max() and mixed["t"][800] < 1_900_000_000
        return on + [("push", "host", first), ("push", "host", older), ("build", 1_900_000_001), ("build", 1_900_000_000),
                     ("push", "host", mixed), ("build", int(mixed["t"].max()) + 1), ("build", 1_900_000_001)]
    if kind == "switched-on-late":
        a = ts_random_stream(W, H, 4000, 74)
        b = ts_jitter(ts_random_stream(W, H, 4000, 75), 76)
        return [("push", "host", ts_cut(a, 0, 2000)), ("unordered_refused",), ("push", "host", ts_cut(a, 2000, 4000))] + _builds(a) + \
               [("reset",), ("unordered", 1)] + _pushes(b, [1000, None]) + _builds(b)
    ev = ts_jitter(ts_random_stream(W, H, 1024 + 1025 + 2048 + 1 + 1023 + 3000, 77), 78)
    how = {"sizes": "host", "nopol": "nopol", "dev": ["dev", "devnopol"], "forward": "host"}[kind]
    return on + _pushes(ev, [1024, 1025, 2048, 1, 1023, None], how) + _builds(ev)


def _s_order_flag(W, H):
    ev = ts_random_stream(W, H, 6000, 81)
    t_end = int(ev["t"][-1]) + 1
    a = ts_cut(ev, 0, 1000)
    bad = ts_cut(ev, 1000, 2000)
    bad = dict(bad, t=bad["t"].copy()); bad["t"][500] = bad["t"][498] - 1                       # violation inside a push
    across = ts_cut(ev, 600, 1600)                                                               # ordered in itself, starts before a's end
    assert across["t"][0] < a["t"][-1]
    later = ts_cut(ev, 2000, 3000)
    fresh = ts_cut(ev, 3000, 6000)
    return [("push", "host", a), ("build", t_end), ("push", "host", bad), ("refused", t_end, TS_UNSUPPORTED), ("reset",),
            ("push", "host", a), ("push", "host", across), ("refused", t_end, TS_UNSUPPORTED),
            ("push", "host", later), ("refused", t_end, TS_UNSUPPORTED),                         # sticky over ordered pushes
            ("reset",), ("push", "host", fresh), ("build", t_end), ("build", int(fresh["t"][1500])), ("fresh", fresh, int(fresh["t"][1500]))]


TS_FWD_BLOCKS = (((20, 20, 10, 10), (100.5, 50.5), 0), ((40, 20, 6, 6), (120.25, 50.75), 1), ((60, 20, 4, 8), (140.5, 60.5), None))
TS_FWD_EXTRA = ((70, 20), (139.5, 60.5))   # one more source next to the 4 x 8 block's point: 33 contributions on two of its pixels


def ts_handbuilt_lut(W, H):
    """Raw pixel -> rectified point table with whole source blocks sent to one point (x0, y0, w, h) -> (u, v): 100, 36 (> the fold
    kernel's 32-entry register list) and exactly 32 contributions per destination, 33 where TS_FWD_EXTRA overlaps; every rejection of
    TimeSurface.cpp:90,95 on the first row; NaN (no contribution) above row 100 elsewhere, a quarter-pixel shift below."""
    lut = np.full((H, W, 2), np.nan)
    yy, xx = np.mgrid[100:H, 0:W]
    lut[100:, :, 0] = xx + 0.25; lut[100:, :, 1] = yy - 0.5
    for (x0, y0, w, h), uv, _ in TS_FWD_BLOCKS:
        lut[y0:y0 + h, x0:x0 + w] = uv
    lut[TS_FWD_EXTRA[0][1], TS_FWD_EXTRA[0][0]] = TS_FWD_EXTRA[1]
    for x, uv in enumerate(((np.nan, 10), (-0.5, 10), (W - 1, 10), (W - 1.5, 10), (W, 10), (10, H - 1), (10, H - 1.5), (10, np.nan), (12, -0.25),
                            (0.0, 0.0), (W - 2.0, H - 2.0))):
        lut[0, x] = uv
    return lut


def _s_fwd_handbuilt(W, H):
    rng = np.random.default_rng(91)
    xs, ys, ps = [], [], []
    for (x0, y0, w, h), _, pol in TS_FWD_BLOCKS:
        for y in range(y0, y0 + h):
            for x in range(x0, x0 + w):
                xs.append(x); ys.append(y); ps.append(int(rng.integers(0, 2)) if pol is None else pol)
    xs.append(TS_FWD_EXTRA[0][0]); ys.append(TS_FWD_EXTRA[0][1]); ps.append(1)
    xs += list(range(11)); ys += [0] * 11; ps += [1, 0] * 5 + [1]
    o = rng.permutation(len(xs))                                           # arrival order is not raster order
    sp = ts_ev(np.array(xs)[o], np.array(ys)[o], np.zeros(len(xs)), np.array(ps)[o])
    bg = ts_random_stream(W, H, 12000, 92)
    bg["y"][:] = np.maximum(bg["y"], 30)                                   # keeps the first row and the blocks to the hand-placed events
    ev = ts_cat(bg, sp)
    ev["t"][bg["t"].size:] = bg["t"][-1] + 1 + np.arange(len(xs)) * 50     # newest: decay close to 1, |sum| far beyond 1
    return _pushes(ev, [5000, None]) + [("build", int(ev["t"][-1]) + 1), ("build", int(ev["t"][-40])), ("build", int(ev["t"][-1]) + 1)]


def _s_evict(W, H):
    """Five pushes of 1.5 M events into the 4 Mi log: folds at the third and at the fifth push (back on the first buffer set)."""
    rng = np.random.default_rng(5)
    n_batch, ops, tt = 1_500_000, [], []
    for b in range(5):
        x = rng.integers(0, W, n_batch); y = rng.integers(0, H, n_batch)
        if b > 0:
            x[x < 40] += 40                                                # these pixels' values come from the base grids
        t = 1_000_000_000 + (b * n_batch + np.arange(n_batch)) * 40
        tt.append(t)
        ops.append(("push", "host", ts_ev(x, y, t, rng.integers(0, 2, n_batch))))
    t = np.concatenate(tt)
    r0 = t.size - (n_batch + TS_LOG_CAP // 4)                              # first resident event after the second fold
    big = ts_ev(np.zeros(TS_LOG_CAP // 2 + 1), np.zeros(TS_LOG_CAP // 2 + 1), np.full(TS_LOG_CAP // 2 + 1, int(t[-1]) + 5))
    return ops + [("build", int(t[-1]) + 1000), ("build", int(t[-200_000])), ("build", int(t[r0 + 1])), ("build", int(t[r0])),
                  ("build", int(t[r0 - 1]) + 1), ("refused", int(t[r0 - 1]), TS_UNSUPPORTED), ("refused", int(t[r0 - 21]), TS_UNSUPPORTED),
                  ("refused", int(t[2_000_000]), TS_UNSUPPORTED), ("refused", int(t[0]), TS_UNSUPPORTED),
                  ("push_refused", big, TS_CAPACITY), ("build", int(t[-1]) + 1000)]


def _sc(id, script, size="hkust", cams=(0, 1), lut=None, **prm):
    return dict(id=id, size=size, prm=prm, script=script, cams=cams, lut=lut)


FWD = dict(time_surface_mode=1)
TS_CASES = [
    _sc("bwd-median0", _s_plain, median_blur_kernel_size=0),
    _sc("bwd-median0-pol", _s_plain, median_blur_kernel_size=0, ignore_polarity=0),
    _sc("median2-refused", lambda W, H: [("push", "host", ts_random_stream(W, H, 3000, 12)), ("refused", 2_000_000_000, TS_UNSUPPORTED), ("sync",),
                                         ("refused", 1_003_000_000, TS_UNSUPPORTED), ("reset",), ("push", "host", ts_random_stream(W, H, 3000, 13))],
        median_blur_kernel_size=2),
    _sc("decay-1ms", _s_plain, decay_ms=1.0),
    _sc("decay-1s", _s_plain, decay_ms=1000.0, ignore_polarity=0),
    _sc("qlen-1", lambda W, H: _s_qlen(W, H, 1), max_event_queue_len=1),
    _sc("qlen-2", lambda W, H: _s_qlen(W, H, 2), max_event_queue_len=2),
    _sc("qlen-64", lambda W, H: _s_qlen(W, H, 64), max_event_queue_len=64),
    _sc("t-edges", _s_t_edges),
    _sc("stamp0-offimage-epoch", _s_stamp0_offimage_epoch, ignore_polarity=0),
    _sc("stamp0-offimage-epoch-fwd", _s_stamp0_offimage_epoch, **FWD),
    _sc("dev-push", lambda W, H: _s_dev(W, H, "dev")),
    _sc("dev-push-nopol", lambda W, H: _s_dev(W, H, "devnopol"), ignore_polarity=0),
    _sc("dev-then-host", lambda W, H: _s_dev(W, H, "dev-then-host")),
    _sc("dev-drain-then-build", lambda W, H: _s_dev(W, H, "dev-drain-then-build")),
    _sc("dev-push-fwd", lambda W, H: _s_dev(W, H, "dev"), **FWD),
    _sc("packet-4095-4096", _s_packet, ignore_polarity=0),
    _sc("unord-ties", lambda W, H: _s_unord(W, H, "ties"), ignore_polarity=0),
    _sc("unord-carry-wins-blocks", lambda W, H: _s_unord(W, H, "carry-wins-blocks"), ignore_polarity=0),
    _sc("unord-1024-1025-2048", lambda W, H: _s_unord(W, H, "sizes"), ignore_polarity=0),
    _sc("unord-nopol", lambda W, H: _s_unord(W, H, "nopol"), ignore_polarity=0),
    _sc("unord-dev", lambda W, H: _s_unord(W, H, "dev"), ignore_polarity=0),
    _sc("unord-forward", lambda W, H: _s_unord(W, H, "forward"), ignore_polarity=0, **FWD),
    _sc("unord-switched-on-late", lambda W, H: _s_unord(W, H, "switched-on-late")),
    _sc("order-flag", _s_order_flag),
    _sc("order-flag-fwd", _s_order_flag, **FWD),
    _sc("fwd-handbuilt", _s_fwd_handbuilt, lut=ts_handbuilt_lut, ignore_polarity=0, median_blur_kernel_size=0, **FWD),
    _sc("fwd-handbuilt-median", _s_fwd_handbuilt, lut=ts_handbuilt_lut, ignore_polarity=1, **FWD),
    _sc("size-small", lambda W, H: _s_plain(W, H, n=8000), size="small"),
    _sc("size-small-fwd", lambda W, H: _s_plain(W, H, n=8000), size="small", ignore_polarity=0, **FWD),
    _sc("size-odd", lambda W, H: _s_plain(W, H, n=20000), size="odd", ignore_polarity=0),
    _sc("size-odd-fwd", lambda W, H: _s_plain(W, H, n=20000), size="odd", **FWD),
    _sc("size-dsec-median0", lambda W, H: _s_plain(W, H, n=40000), size="dsec", median_blur_kernel_size=0),
    _sc("evict-T-before-resident", _s_evict, cams=(0,)),
]
TS_CASES = {c["id"]: c for c in TS_CASES}


def ts_case_script(c):
    W, H = TS_SIZES[c["size"]]
    return c["script"](W, H)


def ts_case_params(c, lib):
    p = configs.params_for("dsec" if c["size"] == "dsec" else "hkust", lib)
    for k, v in c["prm"].items():
        setattr(p, k, v)
    return p


def ts_effective(ops):
    """What the reference's eventsCallback queues for the pushes of a script, one stream per segment between resets
    (tests/indep_numpy.py::events_callback_queue; a stream whose stamps never decrease is its own answer: every insertion stops at
    once and back() is the new event)."""
    import indep_numpy as ind
    seg = [[]]
    for op in ops:
        if op[0] == "push":
            seg[-1].append(dict(op[2], p=np.ones_like(op[2]["p"])) if "nopol" in op[1] else op[2])     # pol = NULL queues polarity 1
        elif op[0] == "reset":
            seg.append([])
    out = []
    for s in seg:
        ev = ts_cat(*s) if s else ts_ev([], [], [])
        out.append(ev if np.all(np.diff(ev["t"]) >= 0) else ind.events_callback_queue(ev))
    return out


def ts_host_model(ops):
    """The host-side bookkeeping of ts_push / ts_run_build / drain (host_knows, host_max_t, log folds) replayed over a script: which
    branch every push and build takes, as a list of sets of tags, one per op."""
    knows, hmax, stamps, unordered, dev_seen, tags = True, None, [], False, False, []
    log_n, folds, fold_t = 0, 0, None
    eff = ts_effective(ops)
    seg, pushed = 0, 0
    for op in ops:
        tg = set()
        if op[0] == "push":
            ev, how = op[2], op[1]
            n = ev["t"].size
            if log_n + n > TS_LOG_CAP:
                keep = min(log_n, TS_LOG_CAP // 4)
                fold_t = int(eff[seg]["t"][pushed - keep - 1]); log_n = keep; folds += 1
                tg.add("fold%d" % folds)
            run_max = int(eff[seg]["t"][pushed - 1]) if pushed else None
            dev = how.startswith("dev")
            tg.add(how)
            if unordered:
                tg.add("unordered")
                if pushed == 0:
                    tg.add("scan-empty-carry")
                for b in range(0, n, 1024):
                    blk = ev["t"][b:b + 1024]
                    if run_max is not None and blk.max() < run_max:
                        tg.add("scan-block-older-than-carry")
                    if run_max is not None and b == 0 and blk[0] == run_max:
                        tg.add("scan-tie-with-carry")
                inc = np.maximum.accumulate(ev["t"])
                if np.any(ev["t"][1:] == inc[:-1]):
                    tg.add("scan-tie")
                tg.add("scan-n%d" % n)
            if dev or unordered:
                knows = False
            elif knows:
                if hmax is None or ev["t"][-1] >= hmax:
                    hmax = int(ev["t"][-1])
                else:
                    knows = False
            if not dev and dev_seen:
                tg.add("host-after-dev")
            dev_seen |= dev
            if how.startswith("packet"):
                tg.add("packet-one-copy" if (how == "packet" and n >= 4096) else "packet-four-copies")
            if not unordered:
                if np.any(np.diff(ev["t"]) < 0):
                    tg.add("order-violation-inside")
                elif run_max is not None and ev["t"][0] < run_max:
                    tg.add("order-violation-across")
            pushed += n; log_n += n
            stamps = eff[seg]["t"][:pushed]
        elif op[0] == "sync":
            if not knows and not unordered:
                knows, hmax = True, (int(stamps.max()) if len(stamps) else None)
                tg.add("drain-refreshes-host")
        elif op[0] == "reset":
            knows, hmax, stamps, dev_seen, log_n, fold_t = True, None, [], False, 0, None
            seg += 1; pushed = 0
        elif op[0] == "unordered":
            unordered = bool(op[1])
        elif op[0] in ("build", "refused"):
            T = op[1]
            if log_n == 0:
                tg.add("empty-log")
            fast = knows and (log_n == 0 or T > hmax)
            general = len(stamps) > 0 and T <= int(stamps[-1])
            tg.add("fast" if fast else ("general" if general else "general-launched-as-no-op"))
            assert not (fast and general)
            if knows and hmax is not None and T == hmax:
                tg.add("T==host_max_t")
            if knows and hmax is not None and T == hmax + 1:
                tg.add("T==host_max_t+1")
            if len(stamps) and T == int(stamps[0]):
                tg.add("T==oldest")
            if len(stamps) and np.sum(stamps == T) >= 3:
                tg.add("T==shared-stamp")
            if fold_t is not None:
                tg.add("T<=folded" if T <= fold_t else "T>folded")
                if T == int(stamps[pushed - log_n]):
                    tg.add("T==oldest-resident")
        tags.append(tg)
    return tags
