"""BASELINE.json's full sizes on the GPU: the BENCHMARKED configurations against the oracle (configs[1]: 5 000 events per
frame, 20-frame fusion window, 25 frames; configs[2]: dsec 20 000 events, fusion_radius 1, SmoothTimeSurface, 5-frame window,
7 frames -- bench.parity_block, the same code that fills BENCH.parity), plus size-independent properties: determinism /
idempotence, range and ordering invariants, pipeline-depth invariance, and the Mapping -> Tracking loop (configs[3])."""
import ctypes as C

import numpy as np
import pytest

from esvo_b200 import capi, configs, synth
from util import build_ts_pair, make_backends, rel, scenario

pytestmark = pytest.mark.gpu


def _gpu_backend(product_lib, rig, tweak=None):
    l, r = configs.rig_calibs(rig)
    p = configs.params_for(rig, product_lib)
    if tweak:
        tweak(p)
    return capi.Backend(product_lib, l, r, p)


def _frame(g, s):
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
        g.ts_build(cam, s["t_ts_ns"], want_idx=False, want_ts=False)
    g.set_ts_pair(None, None, s["T_world_left"])
    sd = s["seeds"]
    c = g.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    return c, g.map_download()


def _assert_parity(par):
    assert par["idx_grid_equal"] and par["ts_bytes_equal"] and par["ts_mismatching_pixels"] == 0          # bit-exact integer work
    assert par["accept_set_symmetric_difference"] == 0 and par["disparity_mismatches"] == 0 and par["seeds_compared"] > 0
    assert par["lm_accept_symmetric_difference"] == 0 and par["lm_points_compared"] > 0
    assert par["counters_equal"] and par["map_size_equal"] and par["map_order_equal"] and par["map_checksum_equal"]
    # inverse depth: 1e-4 relative is the north star's tolerance.  The forward-difference LM amplifies rounding differences
    # into different termination points for a handful of flat problems, so the bound is on the mean and on the fraction
    assert par["inv_depth_l1"] <= 1e-6 and par["inv_depth_frac_above_1e-4"] <= 1e-3, par
    assert par["map_inv_depth_l1"] <= 1e-6 and par["map_inv_depth_frac_above_1e-4"] <= 1e-3, par


def test_cfg2_benchmarked_configuration_matches_oracle(product_lib):
    """BASELINE configs[1] exactly as bench.py runs it: 5 000 events per frame, 20-frame window primed, then 5 consecutive
    frames (25 in total) compared stage by stage; then the tracker on the last fused map (configs[3], tracking_hkust.yaml)."""
    import bench
    base = bench.make_workload(seed=10)
    assert base["seeds"]["x"].size == 5000
    par, trk = bench.parity_block(product_lib, base, "hkust", n_check=5, tracking=True)
    print("cfg2 parity:", par)
    assert par["frames_primed"] == 20 and par["frames_checked"] == 5
    _assert_parity(par)
    assert trk["ts_equal"]
    for mode in ("analytical", "numerical"):
        t = trk[mode]
        assert t["stats_equal"] and t["pose_max_abs_diff_vs_oracle"] < 1e-6 and t["translation_rel_diff_vs_oracle"] < 1e-4, t


def test_dense_scene_long_contribution_lists_match_oracle(product_lib):
    """Scene 11 of the synthetic generator is denser (85 k events per frame): single pixels collect several hundred
    contributions over the 20-frame window, which takes the fold's sort-pool path (lists longer than its local array)."""
    import bench
    base = bench.make_workload(seed=11)
    par, _ = bench.parity_block(product_lib, base, "hkust", n_check=2, tracking=False)
    print("scene 11 parity:", par)
    _assert_parity(par)


def test_cfg3_dsec_benchmarked_configuration_matches_oracle(product_lib):
    """SURVEY 8d cfg 3: 640x480 dsec rig, 20 000 events, disparity [0, 80], fusion_radius 1, SmoothTimeSurface, 5-frame window
    (mapping_dsec.yaml): window primed with 5 frames, 2 more compared."""
    import bench
    base = bench.make_workload(seed=3, cfg="cfg3")
    assert base["seeds"]["x"].size == 20000
    par, _ = bench.parity_block(product_lib, base, "dsec", n_check=2, tracking=False)
    print("cfg3 parity:", par)
    assert par["frames_primed"] == 5
    _assert_parity(par)


@pytest.mark.parametrize("rig,n_seeds", [("hkust", 5000), ("dsec", 20000)])
def test_full_size_frame_properties(product_lib, rig, n_seeds):
    """configs[1] (346x260, 5k seeds) and configs[2] (640x480, 20k seeds + fusion)."""
    kw = dict(n_segments=120) if rig == "dsec" else {}
    s = synth.make_stream(rig, seed=3, n_seeds=n_seeds, **kw)
    assert s["seeds"]["x"].size == n_seeds
    g1 = _gpu_backend(product_lib, rig)
    c1, m1 = _frame(g1, s)
    d = g1.get_derived()
    # accounting identities
    assert c1["n_events"] == n_seeds and c1["n_seeds"] <= n_seeds and c1["n_solved"] <= c1["n_seeds"] and c1["n_culled"] <= c1["n_solved"]
    ncand = d["max_disparity"] - d["min_disparity"] + 1
    assert c1["bm_evals"] <= n_seeds * (ncand + 1) and c1["bm_evals"] >= c1["n_seeds"] * 2
    assert c1["lm_evals"] >= c1["n_seeds"] * 3 and c1["lm_evals"] <= c1["n_seeds"] * 30 * 11
    assert c1["n_seeds"] > 0.2 * n_seeds and c1["map_size"] == m1.size > 0
    # map invariants: one element per pixel, inside the image; (regularisation marks rejected points with rho = -1)
    pix = m1["row"].astype(np.int64) * 4096 + m1["col"]
    H, W = g1.H, g1.W
    assert (m1["row"] >= 0).all() and (m1["row"] < H).all() and (m1["col"] >= 0).all() and (m1["col"] < W).all()
    valid = m1["inv_depth"] > -1e-6
    p = g1.params
    assert valid.any()
    assert np.isfinite(m1["inv_depth"]).all() and (m1["variance"][valid] >= 0).all()
    # idempotence / determinism: a second context fed the same inputs produces the same bytes
    g2 = _gpu_backend(product_lib, rig)
    c2, m2 = _frame(g2, s)
    assert c1 == c2 and m1.tobytes() == m2.tobytes()
    # seeds: disparities inside the clipped range, thread-major order is a permutation of accepted events
    sd = s["seeds"]
    seeds, ev = g2.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    assert seeds.size == c1["n_seeds"] and ev == c1["bm_evals"]
    assert (seeds["disp"] >= d["min_disparity"]).all() and (seeds["disp"] <= d["max_disparity"]).all()
    assert (seeds["cost"] <= 0.1).all() and (seeds["cost"] >= -1e-9).all()
    fb = seeds["disp"] / np.where(seeds["inv_depth"] > 0, seeds["inv_depth"], np.nan)
    assert np.nanmax(np.abs(fb - np.nanmedian(fb))) < 1e-6 * np.nanmedian(fb)      # inv_depth = disp / (f b)


def test_pipeline_depth_invariance_full_size(product_lib):
    """Frames processed with 1, 3 and 8 frames in flight give byte-identical maps and counters, and so does one context
    whose depth changes between frames (3, 3, 1, 4: every outstanding ticket is collected before each switch)."""
    s = [synth.make_stream("hkust", seed=4, n_seeds=5000, t_ts=t, history_ms=50.0) for t in (0.50, 0.55, 0.60, 0.65)]
    ref = None
    for schedule in ((1,) * 4, (3,) * 4, (8,) * 4, (3, 3, 1, 4)):
        def tw(p):
            p.max_num_fusion_frames = 3
        g = _gpu_backend(product_lib, "hkust", tweak=tw)
        tickets, got = [], []
        depth = None
        for f, d in zip(s, schedule):
            if d != depth:
                while tickets:
                    m, c = g.results_end(tickets.pop(0)); got.append((c, m.tobytes()))
                depth = d
                g.set_pipeline_depth(depth)
            if len(tickets) >= max(1, depth - 1):
                m, c = g.results_end(tickets.pop(0)); got.append((c, m.tobytes()))
            for cam, side in ((0, "left"), (1, "right")):
                e = f[side]
                g.stage_ts_events(cam, e["x"], e["y"], e["t"], e["p"])
                g.run_ts_build(cam, f["t_ts_ns"])
            T = np.ascontiguousarray(f["T_world_left"], np.float64)
            g._call("set_ts_pair_dev", [C.POINTER(C.c_double)], T.ctypes.data_as(C.POINTER(C.c_double)))
            sd = f["seeds"]
            g.stage_mapping_inputs(sd["x"], sd["y"], sd["t"], f["pose_t"], f["poses"])
            g.run_mapping()
            tickets.append(g.results_begin())
        while tickets:
            m, c = g.results_end(tickets.pop(0)); got.append((c, m.tobytes()))
        if ref is None:
            ref = got
        else:
            assert [a[0] for a in got] == [a[0] for a in ref]
            assert [a[1] for a in got] == [a[1] for a in ref], f"depths {schedule} changed the maps"


def test_mapping_tracking_loop_matches_oracle(oracle_lib, product_lib):
    """configs[3]: mapping at 20 Hz feeds the local map to the tracker, which tracks the following time surfaces
    (RegProblemLM, analytic Jacobian, Huber); the pose of every tracked frame must match the oracle's."""
    def tw(p):
        p.max_num_fusion_frames = 2
    o, g = make_backends("hkust", oracle_lib, product_lib, tweak=tw)
    times = [0.50, 0.55, 0.60]
    poses_o, poses_g = [], []
    T_prev_o = T_prev_g = None
    for k, t in enumerate(times):
        s = scenario("hkust", n_seeds=3000, t_ts=t)
        tl, tr = build_ts_pair(o, s)
        o.ts_reset(0); o.ts_reset(1)
        clouds = []
        for be in (o, g):
            be.set_ts_pair(tl, tr, s["T_world_left"])
            sd = s["seeds"]
            be.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
            m = be.map_download()      # publishPointCloud sends every element of the list (esvo_Mapping.cpp:923-935)
            Tw = s["T_world_left"]
            pw = m["p_cam"] @ Tw[:3, :3].T + Tw[:3, 3]
            clouds.append(pw.astype(np.float32))
        assert clouds[0].shape == clouds[1].shape and clouds[0].shape[0] >= 500
        perr = np.linalg.norm(clouds[0] - clouds[1], axis=1) / np.linalg.norm(clouds[0], axis=1)
        print(f"frame {k}: map points {clouds[0].shape[0]}, rel point error max {perr.max():.2e}, >1e-4: {(perr > 1e-4).sum()}")
        assert (perr < 1e-4).mean() > 0.995
        # track the NEXT time surface against this map, starting from this frame's pose
        s2 = scenario("hkust", n_seeds=1500, t_ts=t + 0.01)
        tl2, _ = build_ts_pair(o, s2)
        o.ts_reset(0); o.ts_reset(1)
        outs = []
        for be, cloud in ((o, clouds[0]), (g, clouds[0])):     # same cloud bytes into both trackers
            c = cloud.copy()
            be.track_srand(1)
            assert be.track_reset(c, s["T_world_left"], s["T_world_left"], tl2) == 0
            T, st = be.track_solve(True)
            outs.append((T, st))
        (To, so), (Tg, sg) = outs
        assert so == sg, (so, sg)
        assert np.abs(To - Tg).max() < 1e-6 * max(1.0, np.abs(To).max()), np.abs(To - Tg).max()
        poses_o.append(To); poses_g.append(Tg)
    assert len(poses_g) == 3


def test_pipeline_depth16_wraps_around(product_lib):
    """20 frames through 16 pipeline slots (slots, window vectors and result buffers get recycled) == strictly sequential."""
    s = [synth.make_stream("hkust", seed=6, n_seeds=800, t_ts=0.50 + 0.01 * k, history_ms=10.0) for k in range(20)]
    ref = None
    for depth in (1, 16):
        def tw(p):
            p.max_num_fusion_frames = 5
        g = _gpu_backend(product_lib, "hkust", tweak=tw)
        g.set_pipeline_depth(depth)
        tickets, got = [], []
        for f in s:
            if len(tickets) >= max(1, depth - 1):
                m, c = g.results_end(tickets.pop(0)); got.append((c, m.tobytes()))
            for cam, side in ((0, "left"), (1, "right")):
                e = f[side]
                g.stage_ts_events(cam, e["x"], e["y"], e["t"], e["p"])
                g.run_ts_build(cam, f["t_ts_ns"])
            T = np.ascontiguousarray(f["T_world_left"], np.float64)
            g._call("set_ts_pair_dev", [C.POINTER(C.c_double)], T.ctypes.data_as(C.POINTER(C.c_double)))
            sd = f["seeds"]
            g.stage_mapping_inputs(sd["x"], sd["y"], sd["t"], f["pose_t"], f["poses"])
            g.run_mapping()
            tickets.append(g.results_begin())
        while tickets:
            m, c = g.results_end(tickets.pop(0)); got.append((c, m.tobytes()))
        assert len(got) == len(s)
        if ref is None:
            ref = got
            assert sum(c["n_fusions"] for c, _ in ref) > 0 and ref[-1][0]["map_size"] > 100
        else:
            assert [a[0] for a in got] == [a[0] for a in ref]
            assert [a[1] for a in got] == [a[1] for a in ref], "depth 16 changed the maps"
