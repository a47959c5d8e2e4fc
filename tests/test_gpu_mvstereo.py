"""SURVEY 8f row 4: the comparison modes of esvo_MVStereo on the device against the oracle --
EventMatcher [26] (esvo_core/src/core/EventMatcher.cpp), vEMP2vDP, DepthFusion::naive_propagation accumulation, and the five
MVStereoMode sequences of esvo_MVStereo::MappingAtTime (esvo_core/src/esvo_MVStereo.cpp:239-520) assembled from the C ABI."""
import numpy as np
import pytest

from esvo_b200 import capi
from util import build_ts_pair, em_problem, make_backends, rel, scenario

pytestmark = pytest.mark.gpu


def _frame(oracle_lib, product_lib, rig, seed=4, t_ts=0.5, backends=None, tweak=None):
    s = scenario(rig, seed=seed, n_seeds=800, t_ts=t_ts)
    o, g = backends or make_backends(rig, oracle_lib, product_lib, tweak=tweak)
    tl, tr = build_ts_pair(o, s)
    o.ts_reset(0); o.ts_reset(1)
    for be in (o, g):
        be.set_ts_pair(tl, tr, s["T_world_left"])
    return s, o, g


def _same_seeds(so, sg):
    assert so.size == sg.size
    assert np.array_equal(so["t_ns"], sg["t_ns"]), "event order differs"
    for f in ("x_left_raw", "x_left", "x_right", "T_world_virtual", "disp", "inv_depth", "cost"):
        assert np.array_equal(so[f], sg[f]), f


def _same_map(mo, mg, tol=1e-9):
    assert mo.size == mg.size and mo.size > 0
    assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"]), "element order differs"
    for f in ("inv_depth", "variance", "residual", "x", "p_cam"):
        assert np.allclose(mo[f], mg[f], rtol=tol, atol=1e-12), f
    assert np.array_equal(mo["age"], mg["age"])


@pytest.mark.parametrize("rig,kw", [("hkust", dict(time_thr=5e-4, epi_thr=1.0, ncc_thr=0.1, patch=(15, 7), num_thread=4)),
                                    ("hkust", dict(time_thr=1e-4, epi_thr=0.5, ncc_thr=0.3, patch=(25, 5), num_thread=3)),
                                    ("dsec", dict(time_thr=5e-4, epi_thr=1.0, ncc_thr=0.15, patch=(15, 7), num_thread=4))])
def test_event_matcher_parity(oracle_lib, product_lib, rig, kw):
    s, o, g = _frame(oracle_lib, product_lib, rig)
    left, right, counts, poses = em_problem(s)
    so, eo = o.em_match(left, right, counts, poses, **kw)
    sg, eg = g.em_match(left, right, counts, poses, **kw)
    print(rig, kw, "matches", so.size, "of", int(counts.sum()), "zncc evaluations", eo)
    assert so.size > 30 and eo == eg
    _same_seeds(so, sg)


def test_event_matcher_edge_cases(oracle_lib, product_lib):
    s, o, g = _frame(oracle_lib, product_lib, "hkust")
    left, right, counts, poses = em_problem(s)
    # no slices / no candidates -> no matches, no error
    for be in (o, g):
        sd, ev = be.em_match(left, right, np.zeros(0, np.int32), np.zeros((0, 16)))
        assert sd.size == 0 and ev == 0
        empty = {k: v[:0] for k, v in right.items()}
        sd, ev = be.em_match(left, empty, counts, poses)
        assert sd.size == 0 and ev == 0
    # a threshold of 1 accepts events whose candidates all failed the warp (min_cost stays 1, first candidate, depth 0 -> rho = inf)
    kw = dict(time_thr=5e-4, epi_thr=1.0, ncc_thr=1.0, patch=(15, 7), num_thread=2)
    so, eo = o.em_match(left, right, counts, poses, **kw)
    sg, eg = g.em_match(left, right, counts, poses, **kw)
    assert eo == eg
    _same_seeds(so, sg)
    # slices that cover fewer events than given: the rest is ignored (esvo_MVStereo.cpp:1010 "a small number of events are ignored")
    so, _ = o.em_match(left, right, counts[:2], poses[:2])
    sg, _ = g.em_match(left, right, counts[:2], poses[:2])
    assert so.size > 0
    _same_seeds(so, sg)


def test_vemp2vdp_and_naive_accumulation_parity(oracle_lib, product_lib):
    """PURE_EVENT_MATCHING (mode 0) over three frames: matcher -> vEMP2vDP -> window -> naive_propagation newest first."""
    o = g = None
    window_o, window_g = [], []
    for k, t_ts in enumerate((0.50, 0.53, 0.56)):
        s, o, g = _frame(oracle_lib, product_lib, "hkust", t_ts=t_ts, backends=(o, g) if o else None)
        left, right, counts, poses = em_problem(s)
        so, _ = o.em_match(left, right, counts, poses)
        sg, _ = g.em_match(left, right, counts, poses)
        _same_seeds(so, sg)
        po, pg = o.seeds_to_points(so), g.seeds_to_points(sg)
        assert np.array_equal(po["row"], pg["row"]) and np.array_equal(po["col"], pg["col"]) and np.array_equal(po["age"], pg["age"])
        for f in ("x", "inv_depth", "variance", "scale2", "nu", "T_world_cam"):
            assert np.array_equal(po[f], pg[f]), f
        assert np.allclose(po["residual"], pg["residual"], rtol=0, atol=1e-9)      # = the matcher's cost of each side
        assert np.allclose(po["p_cam"], pg["p_cam"], rtol=1e-12, atol=0)
        window_o.append(po); window_g.append(pg)
        for be, win in ((o, window_o), (g, window_g)):
            for q, v in enumerate(reversed(win[-2:])):             # maxNumFusionFrames = 2, newest first (esvo_MVStereo.cpp:282-286)
                be.naive_propagate(v, s["T_world_left"], q == 0)
        _same_map(o.map_download(), g.map_download())


def _sgm_points(be, s, disp16, num_disparities=48):
    """The PURE_SEMI_GLOBAL_MATCHING branch between the SGM call and the accumulation (esvo_MVStereo.cpp:320-352):
    createEdgeMask(undistorted events, radius 0) (:1130-1175), x < numDisparities and disp < 0 skipped, var 0, residual 0."""
    sd = s["seeds"]
    lut = be.get_rectify_tables(0)[2]
    c = np.floor(lut[sd["y"].astype(int), sd["x"].astype(int)]).astype(np.int64)
    inside = (c[:, 0] >= 0) & (c[:, 0] < be.W) & (c[:, 1] >= 0) & (c[:, 1] < be.H)
    c = c[inside]
    disp = disp16[c[:, 1], c[:, 0]] / 16.0
    keep = (c[:, 0] >= num_disparities) & (disp >= 0)
    c, disp = c[keep], disp[keep]
    seeds = np.zeros(c.shape[0], capi.SEED_DTYPE)
    seeds["x_left"] = c.astype(np.float64)
    seeds["inv_depth"] = disp / (be.get_derived()["baseline"] * s["Pl00"])
    seeds["T_world_virtual"] = np.asarray(s["T_world_left"], float).ravel()
    pts = be.seeds_to_points(seeds)
    pts["row"], pts["col"] = c[:, 0], c[:, 1]          # DepthPoint dp(x, y): the reference passes (x, y) as (row, col) (:336)
    return pts


def _run_mode(be, mode, s, window, max_frames, disp16=None):
    """One esvo_MVStereo::MappingAtTime (esvo_MVStereo.cpp:239-520) in MVStereoMode `mode` through the granular C ABI."""
    p = be.params
    sd = s["seeds"]
    T = s["T_world_left"]
    if mode == 4:
        window.append(_sgm_points(be, s, disp16))
        del window[:-max_frames]
        for q, v in enumerate(reversed(window)):
            be.naive_propagate(v, T, q == 0)
        return be.map_download()
    if mode in (0, 2):
        left, right, counts, poses = em_problem(s)
        vemp, _ = be.em_match(left, right, counts, poses)
    else:
        vemp, _ = be.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    if mode in (0, 1):
        window.append(be.seeds_to_points(vemp))
        del window[:-max_frames]
        for q, v in enumerate(reversed(window)):
            be.naive_propagate(v, T, q == 0)
        return be.map_download()
    vdp, _ = be.depth_solve(vemp)                                     # :449-453
    cost_thr = p.residual_vis_threshold ** 2 * p.patch_size_x * p.patch_size_y
    vdp = be.depth_cull(vdp, p.stdvar_vis_threshold, cost_thr, p.invdepth_min_range, p.invdepth_max_range)
    window.append(vdp)
    del window[:-max_frames]                                          # CONST_FRAMES (:474-479)
    for q, v in enumerate(reversed(window)):
        be.fuse(v, T, p.fusion_radius, q == 0)                        # :489-493
    be.map_clean(p.stdvar_vis_threshold ** 2, p.age_vis_threshold, p.invdepth_max_range, p.invdepth_min_range)
    if p.regularization:
        be.map_regularize()
    return be.map_download()


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_mvstereo_modes_match_oracle(oracle_lib, product_lib, mode):
    """MVStereoMode 0 PURE_EVENT_MATCHING, 1 PURE_BLOCK_MATCHING, 2 EM_PLUS_ESTIMATION, 3 BM_PLUS_ESTIMATION (= the ESVO mapper)
    over three frames with a two-frame window, product vs oracle."""
    o = g = None
    wo, wg = [], []
    for k, t_ts in enumerate((0.50, 0.53, 0.56)):
        s, o, g = _frame(oracle_lib, product_lib, "hkust", t_ts=t_ts, backends=(o, g) if o else None)
        mo = _run_mode(o, mode, s, wo, 2)
        mg = _run_mode(g, mode, s, wg, 2)
        print("mode", mode, "frame", k, "map", mo.size, mg.size)
        assert mo.size == mg.size and mo.size > 20
        assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"])
        assert np.array_equal(mo["age"], mg["age"])
        if mode in (0, 1):
            _same_map(mo, mg)
        else:
            r = rel(mg["inv_depth"], mo["inv_depth"])
            assert (r < 1e-4).mean() > 0.995 and np.median(r) < 1e-7, (np.median(r), r.max())


def test_mvstereo_sgm_mode_matches_oracle(oracle_lib, product_lib):
    """MVStereoMode 4 PURE_SEMI_GLOBAL_MATCHING: the device SGBM (bit-exact vs cv2, tests/test_gpu_sgbm.py) feeds the product,
    cv2.StereoSGBM itself feeds the oracle; point creation + naive accumulation over three frames."""
    cv2 = pytest.importorskip("cv2")
    from esvo_b200 import configs
    o = g = None
    wo, wg = [], []
    for k, t_ts in enumerate((0.50, 0.53, 0.56)):
        s, o, g = _frame(oracle_lib, product_lib, "hkust", t_ts=t_ts, backends=(o, g) if o else None)
        s = dict(s); s["Pl00"] = configs.rig_arrays("hkust")["left"]["P"][0, 0]
        d_dev = g.sgbm_compute()
        tl, tr = build_ts_pair(o, s); o.ts_reset(0); o.ts_reset(1)
        d_ref = cv2.StereoSGBM_create(0, 48, 11, 8 * 121, 32 * 121, -1, 0, 11).compute(tl, tr)
        assert np.array_equal(d_dev, d_ref)
        mo = _run_mode(o, 4, s, wo, 2, d_ref)
        mg = _run_mode(g, 4, s, wg, 2, d_dev)
        print("mode 4 frame", k, "points", wo[-1].size, "map", mo.size)
        assert wo[-1].size > 50
        _same_map(mo, mg)
