"""The host half of the multi-view stereo node (esvo_core::MVStereoFrontEnd in include/esvo_b200/esvo_core.hpp, through
examples/mvstereo_node_dump.cpp) against its restatement from the reference (tests/indep_mvstereo.py) on scripted streams,
in every MVStereoMode, with small and UNIX-epoch stamps; the scripted streams reach every rule they are meant to pin; the
system example builds and stops cleanly without a GPU; the rpg rig's product tables against cv2."""
import os
import subprocess

import numpy as np
import pytest

from conftest import has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "esvo_b200", "_build")
W, H = 346, 260
DT = 10_000_000                 # 100 Hz ticks, mapping every 5th
BASES = {"small": 5_000_000, "epoch": 1_600_000_000 * 10**9}
# the stream's features, in ticks (see _script)
RIGHT_GAP = (40, 70)            # no right events: the EM window runs empty ...
RIGHT_SINGLE = 62               # ... but for one event in tick 62's interval: then it holds exactly that one
LEFT_GAP = (80, 100)            # no left events from tick 79's end on: the SGM walk starts one past the newest event
POSE_START = 13.5               # first pose at 135 ms: the first BM windows miss their oldest samples
POSE_AHEAD = (104, 0.49)        # after tick 104's poses the next one is 0.49 s later: no reset
POSE_JUMP = (165, 0.6)          # after tick 165's poses the next one is 0.6 s later: reset
N_TICKS = 240


def _node_kw(mode):
    return dict(mode=mode, pen=15, ts_len=12, em_num=50, half=0.001, denoising=mode == 1, marker=mode == 3)


def _pose(t_ns, base):
    from esvo_b200 import synth
    return synth.pose_at((t_ns - base) * 1e-9)


def _script(base, seed=0):
    """The node's callbacks in the order esvo_MVStereoSystem makes them (DESIGN.md section 5)."""
    rng = np.random.default_rng(seed)
    pose_t, t = [], base + int(POSE_START * DT)
    while t < base + N_TICKS * DT:
        pose_t.append(t)
        t += 1_000_000
        for k, jump in (POSE_AHEAD, POSE_JUMP):
            if pose_t[-1] < base + k * DT <= t:
                t = pose_t[-1] + int(jump * 1e9)
    ops, p = [], 0
    for k in range(N_TICKS):
        tk = base + k * DT
        for side, gap in (("L", LEFT_GAP), ("R", RIGHT_GAP)):
            n = 0 if (k == 0 or gap[0] <= k < gap[1]) else int(rng.integers(20, 40))
            if side == "R" and k == RIGHT_SINGLE:
                n = 1
            ts = np.sort(rng.integers(tk - DT, tk, n)).astype(np.int64)
            if side == "L" and k == LEFT_GAP[0] - 1 and n:
                ts[-1] = tk - 1000                    # the newest left event sits 1 us before the tick
            lo, hi = (150, 162) if side == "L" else (0, W)   # left events cluster, so that the 3x3 median keeps some of them
            ops.append((side, dict(x=rng.integers(lo, hi, n).astype(np.uint16), y=rng.integers(lo - 50, hi - 50 if side == "L" else H, n).astype(np.uint16),
                                   t=ts, p=rng.integers(0, 2, n).astype(np.uint8))))
        ops.append(("TS", tk))
        if k % 5 == 0:
            while p < len(pose_t) and pose_t[p] <= tk:
                ops.append(("POSE", pose_t[p], _pose(pose_t[p], base)))
                p += 1
            ops.append(("PASS",))
    return ops


def _dump(tmp_path, node_kw, ops):
    import indep_mvstereo as imv
    exe = str(tmp_path / "mvstereo_node_dump")
    subprocess.check_call(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "mvstereo_node_dump.cpp"),
                           "-o", exe])
    imv.write_script(tmp_path / "s.bin", W, H, node_kw, ops)
    p = subprocess.run([exe, str(tmp_path / "s.bin"), str(tmp_path / "o.bin")], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return imv.parse_dump(tmp_path / "o.bin", len(ops))


@pytest.mark.parametrize("base", list(BASES))
@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
def test_node_host_logic_matches_restatement(tmp_path, mode, base):
    """Reset decisions of every callback; per pass the gate, dataTransferring's result, the skip, the observation and its
    pose, the EM bounds, every selected event (EM left / right, SGM, BM window, BM denoised) and the pose samples."""
    import indep_mvstereo as imv
    ops = _script(BASES[base])
    kw = _node_kw(mode)
    cpp, py = _dump(tmp_path, kw, ops), imv.run_script(W, H, kw, ops)
    n_pass = 0
    for i, (c, q) in enumerate(zip(cpp, py)):
        tag = f"op {i} {ops[i][0]}"
        assert c["kind"] == q["kind"] and c["reset"] == q["reset"], tag
        if c["kind"] != 4:
            continue
        n_pass += 1
        for key in ("gated", "transferred", "has_obs", "t_obs", "t_low", "t_up"):
            assert c[key] == q[key], (tag, key, c[key], q[key])
        assert np.abs(c["T_obs"] - q["T_obs"]).max() <= 1e-12, tag
        for key in ("em_left", "em_right", "sgm", "window", "close"):
            assert np.array_equal(c[key], q[key]), (tag, key, c[key].size, q[key].size)
        assert np.array_equal(c["st_t"], q["st_t"]), tag
        assert c["st_T"].shape == q["st_T"].shape and (c["st_T"].size == 0 or np.abs(c["st_T"] - q["st_T"]).max() <= 1e-12), tag
    assert n_pass == N_TICKS // 5


def test_scripted_streams_reach_every_rule():
    """The scripts above reach: every mode with an observation; the `<=` extra event of the EM window; the EM window's
    `return false` with an observation loaded, on a window with exactly one event (the reference's rule) and with none; the SGM walk from one past the newest event; a getPoseAt miss that skips a
    pose sample; a pose 0.49 s ahead that does not reset and a 0.6 s jump that does; the gate and the no-pose skip."""
    import indep_mvstereo as imv
    for base in BASES.values():
        ops = _script(base)
        pose_ops = [i for i, o in enumerate(ops) if o[0] == "POSE"]
        for mode in range(5):
            kw = _node_kw(mode)
            out = imv.run_script(W, H, kw, ops)
            passes = [d for d in out if d["kind"] == 4]
            assert sum(d["has_obs"] for d in passes) >= 20, mode
            assert any(not d["gated"] for d in passes) and any(d["gated"] and not d["has_obs"] for d in passes), mode
            if mode in (0, 2):
                assert any(d["em_left"].size == kw["em_num"] + 1 for d in passes), mode
                for n_right in (0, 1):       # `return false` on no event (undefined in the reference) and on exactly one
                    assert any(d["has_obs"] and not d["transferred"] and d["em_right_window"] == n_right for d in passes), (mode, n_right)
            if mode == 4:
                assert any(d["sgm_past_end"] and d["sgm"].size > 0 for d in passes)
            if mode in (1, 3):
                assert any(d["pose_miss"] for d in passes), mode
                assert any(0 < d["close"].size < d["window"].size for d in passes), mode
            stamps = [ops[i][1] for i in pose_ops]
            gaps = {round((b - a) * 1e-9, 3): out[pose_ops[j + 1]]["reset"] for j, (a, b) in enumerate(zip(stamps, stamps[1:])) if b - a > DT}
            assert gaps == {0.49: False, 0.6: True}, gaps


def test_mvstereo_system_builds_and_fails_cleanly_without_gpu(product_lib, tmp_path):
    import indep_mvstereo as imv
    from esvo_b200 import capi, configs
    exe = str(tmp_path / "mvstereo_system")
    subprocess.check_call(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "mvstereo_system.cpp"),
                           "-L" + BUILD, "-lesvo_b200", "-Wl,-rpath," + BUILD, "-o", exe])
    if has_gpu():
        return
    e = dict(x=np.zeros(1, np.uint16), y=np.zeros(1, np.uint16), t=np.ones(1, np.int64), p=np.zeros(1, np.uint8))
    l, r = configs.rig_calibs("rpg")
    imv.write_scenario(tmp_path / "s.bin", l, r, configs.mvstereo_params_for("rpg", product_lib), DT, DT, 3, configs.mvstereo_config("rpg"),
                       e, e, [DT], np.eye(4).reshape(1, 16))
    p = subprocess.run([exe, str(tmp_path / "s.bin"), str(tmp_path / "r.bin")], capture_output=True, text=True)
    assert p.returncode == 2 and "no CPU fallback" in p.stdout, p.stdout + p.stderr
    (tmp_path / "bad.bin").write_bytes(b"\0" * 8)
    assert subprocess.run([exe, str(tmp_path / "bad.bin"), str(tmp_path / "r.bin")], capture_output=True).returncode == 65


def test_rpg_product_tables_match_cv2(product_lib):
    """calib/rpg: the product's rectification tables against cv2, as tests/test_product_tables_cv2.py pins the other rigs."""
    cv2 = pytest.importorskip("cv2")
    from esvo_b200 import capi, configs
    arr = configs.rig_arrays("rpg")
    Wr, Hr = arr["width"], arr["height"]
    for cal, side in zip(configs.rig_calibs("rpg"), ("left", "right")):
        c = arr[side]
        m1, m2, lut, mask = capi.compute_rectify_tables(product_lib, cal)
        raw = np.stack(np.meshgrid(np.arange(Wr, dtype=np.float32), np.arange(Hr, dtype=np.float32)), -1).reshape(-1, 1, 2)
        r1, r2 = cv2.initUndistortRectifyMap(c["K"], c["D"], c["R"], c["P"], (Wr, Hr), cv2.CV_32FC1)
        und = cv2.undistortPoints(raw, c["K"], c["D"], R=c["R"], P=c["P"]).reshape(Hr, Wr, 2)
        assert np.abs(m1 - r1).max() <= 1e-5 and np.abs(m2 - r2).max() <= 1e-5
        q = lambda a: np.rint(a.astype(np.float32) * np.float32(32)).astype(np.int64)
        assert np.array_equal(q(m1), q(r1)) and np.array_equal(q(m2), q(r2))
        assert np.array_equal(lut, und.astype(np.float64))
        mk = (cv2.remap(np.ones((Hr, Wr), np.float32), r1, r2, cv2.INTER_LINEAR) > 0.999).astype(np.uint8) * 255
        assert np.array_equal(mask, mk)


def test_mvstereo_params_follow_the_table(product_lib):
    """mvstereo_params_for carries the table's back-end keys into esvo_params, per dataset."""
    from esvo_b200 import capi, configs
    for name in ("rpg", "upenn"):
        c, p = configs.mvstereo_config(name), configs.mvstereo_params_for(name, product_lib)
        assert (p.invdepth_min_range, p.invdepth_max_range, p.stdvar_vis_threshold) == (c["invDepth_min_range"], c["invDepth_max_range"], c["stdVar_vis_threshold"])
        assert p.fusion_strategy == (capi.FUSION_CONST_FRAMES if c["FUSION_STRATEGY"] == "CONST_FRAMES" else capi.FUSION_CONST_POINTS)
        assert (p.max_num_fusion_frames, p.max_num_fusion_points, p.regularization) == (c["maxNumFusionFrames"], c["maxNumFusionPoints"], int(c["Regularization"]))
