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
