"""CPU pins of the map side over util.MAP_CASES: the oracle's esvo_fuse / esvo_map_regularize against the scalar restatement
of the reference in tests/indep_fusion.py, for both norms, at the image edge, on both arms of every fast-path guard of the
device's Student-t update, on the l2 variance floor and with decisions placed exactly on their thresholds."""
import numpy as np
import pytest

import indep_fusion as inf
from esvo_b200 import capi, configs
from util import MAP_CASES, MAP_F64, THR_KINDS, bits_equal, map_params, map_point, map_round1, map_round2, map_vec, stack_points

W, H = 346, 260
REG = dict(radius=5, min_nb=8, min_close=8)       # the hkust yaml


def _pl():
    return configs.rig_arrays("hkust")["left"]["P"]


def _oracle(oracle_lib, c, **kw):
    l, r = configs.rig_calibs("hkust")
    p = map_params(c, oracle_lib)
    for k, v in kw.items():
        setattr(p, k, v)
    return capi.Backend(oracle_lib, l, r, p)


def _norm(c):
    return "l2" if c["norm"] == "l2" else "Tdist"


def grid_vs_map_exact(grid, m, tag):
    """The restatement's grid against a downloaded oracle map: order, rows / cols, ages exact; values within 1e-12 (NaN
    where the other is NaN).  Returns the number of f64 values that differ in any bit."""
    assert len(grid.elements) == m.size, (tag, len(grid.elements), m.size)
    assert [e.row for e in grid.elements] == m["row"].tolist() and [e.col for e in grid.elements] == m["col"].tolist(), tag
    assert [e.age for e in grid.elements] == m["age"].tolist(), tag + ": ages"
    get = dict(inv_depth=lambda e: e.rho, scale2=lambda e: e.s2, nu=lambda e: e.nu, variance=lambda e: e.var,
               residual=lambda e: e.res, x=lambda e: e.x)
    ndiff = 0
    for f in MAP_F64:
        a = np.array([get[f](e) for e in grid.elements], np.float64).reshape(m[f].shape)
        assert np.allclose(a, m[f], rtol=1e-12, atol=1e-300, equal_nan=True), (tag, f)
        ndiff += int((~bits_equal(a, m[f])).sum())
    pc = np.array([e.p_cam for e in grid.elements], np.float64).reshape(-1, 3)
    fin = np.isfinite(pc)
    assert np.array_equal(fin, np.isfinite(m["p_cam"])) and np.allclose(pc[fin], m["p_cam"][fin], rtol=1e-9, atol=1e-12), tag
    return ndiff


def run_case(oracle_lib, c, stats=None, per_point=None):
    """Both rounds of case c on the oracle and the restatement, compared after each.  per_point (list, optional) receives
    the branch the restatement took for each round-2 point (one-point vectors, replayed in order)."""
    Pl = _pl()
    o = _oracle(oracle_lib, c)
    pts, T = map_round1(c, Pl)
    grid = inf.Grid(H, W)
    nf_o = o.fuse(pts, T, c["radius"], True)
    nf_p = inf.fuse_vector(grid, map_vec(pts), T, Pl, W, H, c["radius"], stats, norm=_norm(c))
    m1 = o.map_download()
    assert nf_o == nf_p, (c["id"], nf_o, nf_p)
    nd = grid_vs_map_exact(grid, m1, c["id"] + " round 1")
    p2 = map_round2(c, m1, Pl)
    if p2 is None:
        return nd, m1.size
    if c["r2"] == "regmap":
        o.map_regularize()
        grid = inf.regularize(grid, REG["radius"], REG["min_nb"], REG["min_close"], literal=False, norm=_norm(c))
        assert (o.map_download()["inv_depth"] == -1.0).all()
    nf_o = o.fuse(p2, T, c["radius"], False)
    nf_p = 0
    for q in map_vec(p2):
        st = {}
        nf_p += inf.fuse_vector(grid, [q], T, Pl, W, H, c["radius"], st, norm=_norm(c))
        if stats is not None:
            for k, v in st.items():
                stats[k] = stats.get(k, 0) + v
        if per_point is not None:
            per_point.append(st)
    assert nf_o == nf_p, (c["id"], "round 2", nf_o, nf_p)
    m2 = o.map_download()
    return nd + grid_vs_map_exact(grid, m2, c["id"] + " round 2"), m1.size + m2.size


@pytest.mark.parametrize("cid", list(MAP_CASES))
def test_map_case_oracle_vs_restatement(oracle_lib, cid):
    """Element order, rows / cols, ages, fusion counts and every decision exact; values within 1e-12 (the number of values
    that differ in any bit is printed)."""
    stats = {}
    nd, n = run_case(oracle_lib, MAP_CASES[cid], stats)
    print(f"[{cid}] {n} elements compared, {nd} f64 values not bit-identical; branches {stats}")
    assert nd == 0, (cid, nd)


def _case_keys(st):
    return {k for k in ("fuse", "keep", "occluded", "replace", "create") if st.get(k)}


# the decision each threshold contribution must take (round 2 of the "thr" cases); one ulp across a threshold flips it
THR_EXPECT = {
    "Tdist": {("map2s", -1): "fuse", ("map2s", 0): "keep", ("map2s", 1): "keep",
              ("prop2s", -1): "fuse", ("prop2s", 0): "occluded", ("prop2s", 1): "occluded",
              ("occl", -1): "occluded", ("occl", 0): "keep", ("occl", 1): "fuse",
              ("chi", -1): "fuse", ("chi", 0): "fuse", ("chi", 1): "fuse",
              ("tie", "eq"): "keep", ("tie", "var"): "keep", ("tie", "res"): "keep", ("tie", "both"): "replace"},
    "l2": {("map2s", -1): "keep", ("map2s", 0): "keep", ("map2s", 1): "keep",
           ("prop2s", -1): "occluded", ("prop2s", 0): "occluded", ("prop2s", 1): "occluded",
           ("occl", -1): "occluded", ("occl", 0): "keep", ("occl", 1): "keep",
           ("chi", -1): "fuse", ("chi", 0): "keep", ("chi", 1): "keep",
           ("tie", "eq"): "keep", ("tie", "var"): "keep", ("tie", "res"): "keep", ("tie", "both"): "replace"},
}


def test_map_cases_cover_every_fold_branch(oracle_lib):
    """Over the whole table the restatement takes every branch of fold_apply: create / fuse / occluded / replace / keep and
    the "new point" update, both arms of each fast-path guard (S vs 1e-200 and 1e200, nu_u vs 2 and 1e15, the variance
    range of the sqrt_nr switch), nu_u == 2, denormal scales, a NaN compatibility test, the l2 floor in the propagation and
    in the update, points outside the image, a NaN re-projection and points behind the camera.  Each threshold contribution
    of the "thr" cases takes the decision THR_EXPECT names: both outcomes at every threshold."""
    stats = {}
    for cid, c in MAP_CASES.items():
        per = []
        run_case(oracle_lib, c, stats, per)
        if c["r2"] == "thr":
            got = {kind: _case_keys(st) for kind, st in zip(THR_KINDS, per)}
            for kind, exp in THR_EXPECT[_norm(c)].items():
                assert got[kind] == {exp}, (cid, kind, got[kind], per[THR_KINDS.index(kind)])
    print("branch counts over MAP_CASES:", dict(sorted(stats.items())))
    need = ("create", "fuse", "occluded", "replace", "keep", "new_point", "S_lo", "S_ok_lo", "S_hi", "S_ok_hi", "nu_le2",
            "nu_ok_lo", "nu_big", "nu_ok_hi", "nu_eq2", "s2_denormal", "fast", "slow", "fast_var_in", "fast_var_out",
            "compat_nan", "l2_floor_prop", "l2_floor_fuse", "outside", "nan_reprojection", "behind")
    missing = [k for k in need if not stats.get(k)]
    assert not missing, (missing, stats)
    assert stats["fast"] > 20000, stats


def dense_map(Pl, norm, seed=1):
    """A dense hand-built map for the regularisation: one point per 2 x 2 block over two 64 x 50 corners of the image (top
    left: rows / columns below, at and above each radius; bottom right: the last row and column; the splats of fusion
    radius 0 tile them), inverse depths on two smooth surfaces with outliers, Student-t scales 1e-4 .. 1e-2, and rejected
    (rho = -1, behind the camera) blocks."""
    rng = np.random.default_rng(seed)
    qs = []
    blocks = [(by, bx) for by in range(0, 50, 2) for bx in range(0, 64, 2)] + \
             [(by, bx) for by in range(H - 50, H, 2) for bx in range(W - 64, W, 2)]
    for by, bx in blocks:
        k = rng.random()
        if k < 0.25:
            continue                                                     # empty block
        if k < 0.32:
            qs.append(map_point(Pl, bx + 0.5, by + 0.5, -1.0, s2=1e-4, nu=4.0, var=2e-4, exact=False))
            continue
        rho = (0.5 + 0.0004 * bx) if (bx // 40 + by // 40) % 3 else 0.9 + 0.0003 * by
        if rng.random() < 0.1:
            rho *= 1.3                                                   # an outlier: not close to its neighbours
        s2 = 10 ** rng.uniform(-4, -2) * (0.1 if rng.random() < 0.3 else 1.0)
        qs.append(map_point(Pl, bx + rng.uniform(0.05, 0.95), by + rng.uniform(0.05, 0.95), rho * (1 + 0.003 * rng.standard_normal()),
                            s2=s2, nu=2.1897, var=s2 * 2.1897 / 0.1897 if norm != "l2" else s2 * 3, exact=False))
    pts = stack_points(qs)
    return pts


REG_RADII = (0, 1, 2, 3, 5, 7, 20)
REG_COUNTS = ((0, 0), (8, 8), (32, 32))


@pytest.mark.parametrize("norm", ["tdist", "l2"])
def test_regularisation_oracle_vs_restatement(oracle_lib, norm):
    """DepthRegularization::apply at reg_radius 0 .. 20 and min_nb / min_close 0 / 0, 8 / 8, 32 / 32, on a dense hand-built
    map, Tdist and l2: the oracle's inverse depths against the restatement's within 1e-12, the rejected set exact."""
    Pl = _pl()
    c = dict(norm=norm, radius=0)
    pts = dense_map(Pl, norm)
    nd = 0
    for radius in REG_RADII:
        for mn, mc in (REG_COUNTS if radius < 20 else REG_COUNTS[1:2]):
            o = _oracle(oracle_lib, c, reg_radius=radius, reg_min_neighbours=mn, reg_min_close_neighbours=mc)
            o.fuse(pts, np.eye(4), 0, True)
            grid = inf.Grid(H, W)
            inf.fuse_vector(grid, map_vec(pts), np.eye(4), Pl, W, H, 0, norm=_norm(c))
            o.map_regularize()
            g2 = inf.regularize(grid, radius, mn, mc, literal=False, norm=_norm(c))
            m = o.map_download()
            a = np.array([e.rho for e in g2.elements])
            assert m.size == a.size and np.array_equal(m["inv_depth"] == -1.0, a == -1.0), (norm, radius, mn, mc)
            assert np.allclose(a, m["inv_depth"], rtol=1e-12, atol=0), (norm, radius, mn, mc)
            nd += int((~bits_equal(a, m["inv_depth"])).sum())
            print(f"[reg {norm} r={radius} {mn}/{mc}] {m.size} elements, {(a != -1.0).sum()} kept")
    print(f"[reg {norm}] inverse depths not bit-identical to the restatement: {nd}")
    assert nd == 0
