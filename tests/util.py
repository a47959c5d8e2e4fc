"""Shared helpers for the parity tests: one synthetic scenario, two backends fed identical inputs."""
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
