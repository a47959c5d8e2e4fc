"""The multi-view stereo system (include/esvo_b200/esvo_mvstereo_system.hpp, examples/mvstereo_system.cpp) on the GPU, in all
five MVStereoModes, on an rpg-shaped and an upenn-shaped (equidistant) synthetic stream with the trajectory of synth.pose_at
as the ground-truth pose stream: the same stream three ways (the C++ system on the product, the restatement
tests/indep_mvstereo.py on the product and on the oracle), the product against the oracle at every mapping tick at the
MVStereo parity bar of tests/test_gpu_mvstereo.py, and the final map's inverse depth against the scene's."""
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "esvo_b200", "_build")
DT_NS = 10_000_000            # 100 Hz ticks; mapping_rate_hz 20: every 5th tick maps
DURATION_S = 0.8
POSE_DT_NS = 1_000_000        # a 1 kHz ground-truth pose stream
# synth.make_stream arguments: scenes at the depths each rig's yaml maps (inverse-depth range rpg 0.2-2, upenn 0.16-1),
# trajectory at scale 1; the upenn events are distorted with the rig's own equidistant model
STREAMS = {"rpg": dict(depth_range=(0.8, 3.0), n_segments=40), "upenn": dict(depth_range=(1.2, 4.0), n_segments=40)}
# Median relative inverse-depth error of the final map against the synthetic scene, per rig and mode, measured on an
# H100 80GB HBM3 at 700 W (rpg 0.032 0.038 0.250 0.033 0.043, upenn 0.060 0.048 0.021 0.016 0.044 for modes 0-4); the
# bounds are 1.5x those.  rpg mode 2 is the rpg yaml's Regularization on a sparse map (438 points after the 0.015 std-dev cull):
# without it the same run on the oracle has a median of 0.011.
QUALITY = {"rpg": {0: 0.048, 1: 0.057, 2: 0.38, 3: 0.05, 4: 0.065}, "upenn": {0: 0.09, 1: 0.073, 2: 0.033, 3: 0.024, 4: 0.066}}
# Product against oracle over a whole stream.  Modes 0 (EM) and 4 (SGM) are compared end to end: the bar of
# tests/test_gpu_mvstereo.py at every mapping tick (element order, rows / cols / ages exact, values within 1e-9).  In modes 1-3
# an end-to-end comparison amplifies legitimate ties.  The block matcher's cost agrees with the oracle's to ~1e-16, not to the bit
# (the ZNCC sums run in another order), and the naive propagation keeps a point only for a strictly smaller residual.  So two
# seeds with equal inverse depth that the product scores with the very same cost, and the oracle 5.5e-17 apart, pick
# different winners (rpg mode 1, tick 35: 2 of 846 elements), and later frames build
# on that pixel.  The LM's own 1e-4 tail does the same through the fusion's thresholds.  There each stage is held to its bar
# on identical inputs: the oracle's matcher (and LM) output is checked against the product's at the bar of
# tests/test_gpu_mvstereo.py (event-matcher seeds exact, cost included, measured over both streams on an H100 80GB HBM3 at
# 700 W; block-matching seeds exact but the cost, within 1e-9; LM: the same points per pass, inverse depth within 1e-4
# for >= 99.5 % over the stream), and the product's output is handed on, so every map downstream must meet the end-to-end bar.
SUBSTITUTED = {1: ("bm_match",), 2: ("em_match", "depth_solve"), 3: ("bm_match", "depth_solve")}


def _check_seeds(sg, so, exact_cost):
    """tests/test_gpu_mvstereo.py's matcher bar: the event matcher's seeds are exact, cost included; the block matcher's
    cost is within 1e-9 (it is evaluated from integer moments, DESIGN deviation 1)."""
    assert sg.size == so.size
    assert np.array_equal(so["t_ns"], sg["t_ns"]), "event order differs"
    for f in ("x_left_raw", "x_left", "x_right", "T_world_virtual", "disp", "inv_depth"):
        assert np.array_equal(so[f], sg[f]), f
    if exact_cost:
        assert np.array_equal(sg["cost"], so["cost"]), "cost"
    else:
        assert np.allclose(sg["cost"], so["cost"], rtol=0, atol=1e-9)


def _check_lm(pg, po, rels):
    """The LM bar, per pass: the same points in the same order; their relative inverse-depth differences go to `rels`, of
    which at least 99.5 % must lie within 1e-4 over the stream (a pass of ~90 points would otherwise allow none at all)."""
    assert pg.size == po.size and np.array_equal(pg["row"], po["row"]) and np.array_equal(pg["col"], po["col"])
    rels.append(np.abs(pg["inv_depth"] - po["inv_depth"]) / np.abs(po["inv_depth"]))


def _record(be, names):
    """Keeps the outputs of be's stages `names`, in call order."""
    out = {k: [] for k in names}
    for name in names:
        f = getattr(be, name)
        def w(*a, _f=f, _n=name, **kw):
            r = _f(*a, **kw)
            out[_n].append(r)
            return r
        setattr(be, name, w)
    return out


def _substitute(be, names, product_out, rels):
    """be's stages `names` check their own result against the product's at the stage bar, then return the product's."""
    for name in names:
        f, it = getattr(be, name), iter(product_out[name])
        def w(*a, _f=f, _n=name, _it=it, **kw):
            mine, theirs = _f(*a, **kw), next(_it)
            if _n == "depth_solve":
                _check_lm(theirs[0], mine[0], rels)
            else:
                _check_seeds(theirs[0], mine[0], exact_cost=_n == "em_match")
                assert theirs[1] == mine[1], "matcher evaluations"
            return theirs
        setattr(be, name, w)


def _stream(rig, seed=3):
    from esvo_b200 import synth
    return synth.make_stream(rig, seed=seed, t_ts=DURATION_S + 0.05, history_ms=(DURATION_S + 0.05) * 1e3, n_seeds=10,
                             translation_scale=1.0, rig_model=True, **STREAMS[rig])


def _poses(rig, s):
    """The stamped_pose stream: the left camera's pose, or on rpg (dvs_frame_id "marker") the marker's."""
    import indep_mvstereo as imv
    from esvo_b200 import synth
    t = np.arange(int(s["left"]["t"][0]), s["t_ts_ns"] + 1, POSE_DT_NS, dtype=np.int64)
    M = np.linalg.inv(imv.T_MARKER_CAM) if rig == "rpg" else np.eye(4)
    return t, np.array([(synth.pose_at(v * 1e-9) @ M).ravel() for v in t])


def _backends(rig, oracle_lib, product_lib):
    from esvo_b200 import capi, configs
    l, r = configs.rig_calibs(rig)
    g = capi.Backend(product_lib, l, r, configs.mvstereo_params_for(rig, product_lib))
    o = capi.Backend(oracle_lib, l, r, configs.mvstereo_params_for(rig, oracle_lib))
    for cam in (0, 1):
        o.set_rectify_tables(cam, *g.get_rectify_tables(cam))
    return o, g


def _same_records(a, b, keys):
    assert a.size == b.size
    for key in keys:
        assert np.array_equal(a[key], b[key]), (key, a[key].tolist(), b[key].tolist())


def _depth_error(m, T_world_cam, s, Pl):
    """Per map element, the relative error of its inverse depth against the front-most scene point within 1 px of it."""
    from scipy.spatial import cKDTree
    Ti = np.linalg.inv(T_world_cam)
    pc = s["scene_points"] @ Ti[:3, :3].T + Ti[:3, 3]
    pc = pc[pc[:, 2] > 0.1]
    uv = np.stack([Pl[0, 0] * pc[:, 0] / pc[:, 2] + Pl[0, 2], Pl[1, 1] * pc[:, 1] / pc[:, 2] + Pl[1, 2]], 1)
    tree = cKDTree(uv)
    err = []
    for q in m:
        near = tree.query_ball_point(q["x"], 1.0)
        if near:
            rho = 1.0 / pc[near, 2].min()
            err.append(abs(q["inv_depth"] - rho) / rho)
    return np.array(err)


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("rig", ["rpg", "upenn"])
def test_mvstereo_system_three_ways(oracle_lib, product_lib, tmp_path, rig, mode):
    cv2 = pytest.importorskip("cv2")
    import indep_mvstereo as imv
    from esvo_b200 import configs
    s = _stream(rig)
    pose_t, poses = _poses(rig, s)
    cfg = dict(configs.mvstereo_config(rig), MVStereoMode=mode)
    t0 = s["t_ts_ns"] - int(round(DURATION_S * 1e9)) + DT_NS
    n = int(round(DURATION_S * 1e9 / DT_NS))
    Pl = configs.rig_arrays(rig)["left"]["P"]
    # 1. the C++ system on the product
    exe = str(tmp_path / "mvstereo_system")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "mvstereo_system.cpp"),
                           "-L" + BUILD, "-lesvo_b200", "-Wl,-rpath," + BUILD, "-o", exe])
    l, r = configs.rig_calibs(rig)
    imv.write_scenario(tmp_path / "s.bin", l, r, configs.mvstereo_params_for(rig, product_lib), t0, DT_NS, n, cfg, s["left"], s["right"], pose_t, poses)
    p = subprocess.run([exe, str(tmp_path / "s.bin"), str(tmp_path / "r.bin")], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    print(p.stdout.strip())
    sh, sh_map, stopped, _, _, _ = imv.parse_result(tmp_path / "r.bin")
    assert stopped == 0
    # 2. the restatement on the product: identical
    o, g = _backends(rig, oracle_lib, product_lib)
    staged = _record(g, SUBSTITUTED.get(mode, ()))
    pr, pr_map, pr_maps = imv.System(g, lambda a, b: g.sgbm_compute(), cfg, Pl[0, 0], t0, DT_NS).run(s["left"], s["right"], pose_t, poses, n, True)
    keys = ["tick", "t", "gated", "transferred", "ran", "ok", "published", "stamp", "T_kf"] + list(imv.COUNT_KEYS)
    _same_records(sh, pr, keys)
    assert sh_map.tobytes() == pr_map.tobytes()
    ran = pr[pr["ran"] == 1]
    assert ran.size >= 8 and pr["published"].sum() >= 5, pr[["tick", "ran", "ok", "published"]]
    # 3. the restatement on the oracle: the parity bar at every mapping tick (modes 1-3: stage by stage, see SUBSTITUTED)
    rels = []
    _substitute(o, SUBSTITUTED.get(mode, ()), staged, rels)
    sg = cv2.StereoSGBM_create(0, 48, 11, 968, 3872, -1, 0, 11)
    orr, or_map, or_maps = imv.System(o, lambda a, b: sg.compute(a, b), cfg, Pl[0, 0], t0, DT_NS).run(s["left"], s["right"], pose_t, poses, n, True)
    _same_records(pr, orr, keys)
    if rels:
        r = np.concatenate(rels)
        print(f"{rig} mode {mode}: LM on identical seeds, {r.size} points over {len(rels)} passes, {(r < 1e-4).mean():.4f} within 1e-4, "
              f"worst pass {min((x < 1e-4).mean() for x in rels if x.size):.4f}, largest {r.max():.3g}")
        assert (r < 1e-4).mean() >= 0.995
    assert [k for k, _ in pr_maps] == [k for k, _ in or_maps]
    for (k, mg), (_, mo) in zip(pr_maps + [(-1, pr_map)], or_maps + [(-1, or_map)]):
        assert mg.size == mo.size, k
        assert np.array_equal(mg["row"], mo["row"]) and np.array_equal(mg["col"], mo["col"]) and np.array_equal(mg["age"], mo["age"]), k
        for f in ("inv_depth", "variance", "x", "p_cam"):
            assert np.allclose(mo[f], mg[f], rtol=1e-9, atol=1e-12), (k, f)
        assert np.allclose(mo["residual"], mg["residual"], rtol=0, atol=1e-9), k
    # 4. depth quality of the final map
    last = sh[sh["ran"] == 1][-1]
    err = _depth_error(sh_map, last["T_kf"].reshape(4, 4), s, Pl)
    med = float(np.median(err)) if err.size else float("inf")
    print(f"{rig} mode {mode}: {ran.size} mapping passes, {int(pr['published'].sum())} published, final map {sh_map.size}, "
          f"{err.size} with a scene point within 1 px, median relative inverse-depth error {med:.4f}")
    assert sh_map.size >= 50 and err.size >= 0.4 * sh_map.size and med < QUALITY[rig][mode], (sh_map.size, err.size, med)
