"""The closed stereo-odometry loop (include/esvo_b200/esvo_system.hpp, examples/system_loop.cpp) against its restatement from
the reference nodes (tests/indep_system.py): the tf pose buffer, the loop on the oracle following the ground truth, the
re-initialisation path, and on the GPU the same stream three ways (shim on the product, restatement on the product,
restatement on the oracle)."""
import functools
import os
import struct
import subprocess

import numpy as np
import pytest

from conftest import has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "esvo_b200", "_build")
DT_NS = 10_000_000            # 100 Hz sync ticks
DURATION_S = 1.3              # long enough for the fusion window (20 frames at 20 Hz) to fill and publish in WORKING
INIT_TICK = 10                # first mapping tick with more than 10 time surfaces in the history (esvo_Mapping.cpp:497)
HUGE_BATCH = (0, 10**6)       # examples/system_loop.cpp override: trk_batch_size larger than any map, the tracker never works
# Two synthetic hkust scenes (synth.make_stream arguments), both with the hkust yaml (DESIGN.md section 2):
#  * "dense": the default 80-segment scene at the default speed.  Denoising keeps almost none of the newest 1 000 events
#    (edges move ~0.04 px per ms), so the mapper adds nothing after the SGM start-up: the tracker runs on the start-up map.
#  * "mapping": 7 segments at 0.5-1.2 m, trajectory at twice the speed.  The 1 000 events span ~3 ms and cluster on few
#    edges, so the 3x3 median keeps about a third of them: ~170 seeds per WORKING frame, WORKING maps published from tick 105
#    on and adopted by the tracker.
# Bounds from the oracle loop on a CPU (measured: dense ATE 7.6 mm, rotation 0.39 deg; mapping ATE 28.4 mm against 63.5 mm
# for a camera that stays at the start-up pose, rotation 2.7 deg), with a margin of about 1.4-2.6x.
SCENES = {
    "dense": dict(kw=dict(), speed=1.0, ate_m=0.02, rot_deg=1.0),
    "mapping": dict(kw=dict(n_segments=7, speed=2.0, depth_range=(0.5, 1.2)), speed=2.0, ate_m=0.04, rot_deg=4.0),
}


@functools.lru_cache(maxsize=2)
def _stream(scene="dense", duration_s=DURATION_S, seed=2):
    from esvo_b200 import synth
    return synth.make_stream("hkust", seed=seed, t_ts=duration_s, history_ms=duration_s * 1e3, **SCENES[scene]["kw"])


def _ticks(s, duration_s=DURATION_S):
    t0 = s["t_ts_ns"] - int(round(duration_s * 1e9)) + DT_NS
    return t0, int(round(duration_s * 1e9 / DT_NS))


def _gt(t_ns, speed=1.0):
    from esvo_b200 import synth
    return synth.pose_at(t_ns * 1e-9 * speed)    # hkust: translation scale 1


def _cv2_sgbm():
    cv2 = pytest.importorskip("cv2")
    sg = cv2.StereoSGBM_create(0, 48, 11, 968, 3872, -1, 0, 11)   # esvo_Mapping.cpp:101-108
    return lambda l, r: sg.compute(l, r)


def _oracle(oracle_lib, tweak=None):
    from esvo_b200 import capi, configs
    l, r = configs.rig_calibs("hkust")
    p = configs.params_for("hkust", oracle_lib)
    if tweak:
        tweak(p)
    return capi.Backend(oracle_lib, l, r, p)


def _init_stamp(maps):
    ok = maps[(maps["ran"] == 1) & (maps["ok"] == 1)]
    return int(ok[0]["stamp"]), int(ok[0]["tick"])


# ---------------------------------------------------------------- pose buffer (tf restatement)
def _pose_buffer_cpp(tmp_path, stamps, poses, queries):
    exe = str(tmp_path / "pose_buffer_dump")
    subprocess.check_call(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "pose_buffer_dump.cpp"),
                           "-o", exe])
    inp, outp = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(struct.pack("<i", len(stamps))); f.write(np.asarray(stamps, np.int64).tobytes())
        f.write(np.ascontiguousarray(poses, np.float64).tobytes())
        f.write(struct.pack("<i", len(queries))); f.write(np.asarray(queries, np.int64).tobytes())
    p = subprocess.run([exe, str(inp), str(outp)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    raw = open(outp, "rb").read()
    rec = np.frombuffer(raw, np.dtype([("found", "<i4"), ("T", "<f8", (16,))]), len(queries))
    return rec["found"].astype(bool), rec["T"].reshape(-1, 4, 4), struct.unpack_from("<i", raw, rec.nbytes)[0]


def test_pose_buffer_cpp_python_scipy(tmp_path):
    """esvo::PoseBuffer and indep_system.PoseBuffer agree at, between and outside the stamps; between stamps both equal a
    translation lerp and scipy's Slerp of the stored rotations."""
    from scipy.spatial.transform import Rotation, Slerp
    import indep_system as isy
    rng = np.random.default_rng(5)
    stamps = np.sort(rng.choice(np.arange(1, 400), 40, replace=False)).astype(np.int64) * 7_000_001 + 1_600_000_000 * 10**9
    poses = []
    for i, t in enumerate(stamps):
        T = _gt(int(t) - 1_600_000_000 * 10**9)
        if i % 3 == 0:                            # large rotations: the negative-trace branch of Quaterniond(Matrix3d)
            T[:3, :3] = Rotation.from_rotvec(rng.normal(size=3) * 2.5).as_matrix() @ T[:3, :3]
        T[:3, 3] += rng.normal(size=3)
        poses.append(T)
    poses = np.array(poses)
    order = rng.permutation(stamps.size)          # insertion order does not matter
    ins_t = list(stamps[order]) + [stamps[4]]     # a second pose for a stored stamp is refused
    ins_T = list(poses[order]) + [np.eye(4)]
    between = [int(a + (b - a) * f) for a, b, f in zip(stamps[:-1], stamps[1:], rng.uniform(0.01, 0.99, stamps.size - 1))]
    queries = list(stamps) + between + [int(stamps[0]) - 1, int(stamps[-1]) + 1, 1, 0]
    found, Tc, size = _pose_buffer_cpp(tmp_path, ins_t, np.array(ins_T).reshape(-1, 16), queries)
    buf = isy.PoseBuffer()
    for t, T in zip(ins_t, ins_T):
        buf.set_transform(t, T)
    assert size == stamps.size == len(buf.t)
    n_s, n_b = stamps.size, len(between)
    Tp = [buf.lookup(q) for q in queries]
    assert found.tolist() == [T is not None for T in Tp] == [True] * (n_s + n_b) + [False, False, False, True]
    stored = []
    for i in range(n_s):                           # exact stamps: the stored pose after the quaternion round trip, bit for bit
        R = isy.rot_from_quat(isy.quat_from_rot(poses[i][:3, :3]))
        assert np.array_equal(Tc[i], Tp[i]) and np.array_equal(Tc[i][:3, :3], R) and np.array_equal(Tc[i][:3, 3], poses[i][:3, 3])
        assert np.abs(R - poses[i][:3, :3]).max() < 1e-15 * 10
        stored.append(R)
    assert np.array_equal(Tc[-1], Tc[n_s - 1])     # stamp 0: the latest
    sl = Slerp((stamps - stamps[0]).astype(float), Rotation.from_matrix(np.array(stored)))   # epoch stamps do not fit a double
    for j, t in enumerate(between):                # between stamps: lerp + slerp
        i = int(np.searchsorted(stamps, t)) - 1
        r = (t - stamps[i]) / (stamps[i + 1] - stamps[i])
        Rs = sl([float(t - stamps[0])]).as_matrix()[0]
        ts = (1 - r) * poses[i][:3, 3] + r * poses[i + 1][:3, 3]
        for T in (Tc[n_s + j], Tp[n_s + j]):
            assert np.abs(T[:3, :3] - Rs).max() < 1e-12 and np.abs(T[:3, 3] - ts).max() < 1e-12, (j, np.abs(T[:3, :3] - Rs).max())
        assert np.abs(Tc[n_s + j] - Tp[n_s + j]).max() < 1e-12
    # a one-entry buffer answers only at its own stamp
    found1, T1, _ = _pose_buffer_cpp(tmp_path, [stamps[3]], poses[3].reshape(1, 16), [stamps[3], stamps[3] - 1, stamps[3] + 1])
    assert found1.tolist() == [True, False, False] and np.array_equal(T1[0][:3, 3], poses[3][:3, 3])
    one = isy.PoseBuffer(); one.set_transform(stamps[3], poses[3])
    assert one.lookup(stamps[3]) is not None and one.lookup(stamps[3] - 1) is None and one.lookup(stamps[3] + 1) is None
    # the 100 s cache: entries older than the newest minus 100 s are dropped
    found2, _, size2 = _pose_buffer_cpp(tmp_path, [10**9, 2 * 10**9, 150 * 10**9], np.tile(np.eye(4).ravel(), 3), [10**9, 2 * 10**9])
    assert size2 == 1 and not found2.any()


# ---------------------------------------------------------------- the loop on the oracle (CPU)
def _check_follows_gt(ticks, maps, m, scene, tag):
    """SGM start-up at tick 10, WORKING from the next tracker pass, a pose at every later tick, ATE and rotation error under
    the scene's bounds; on the "mapping" scene also real mapping work, non-empty WORKING publishes and a non-empty map."""
    import indep_system as isy
    sc = SCENES[scene]
    t_align, tick0 = _init_stamp(maps)
    assert tick0 == INIT_TICK and maps[maps["tick"] == INIT_TICK]["n_sgm_points"][0] >= 500, tag
    st = ticks["status"]
    assert (st[: INIT_TICK + 1] == 0).all() and (ticks["has_pose"][: INIT_TICK + 1] == 0).all(), tag
    assert (st[INIT_TICK + 1:] == 1).all(), (tag, st.tolist())      # WORKING from the next tracker pass on
    assert (ticks["has_pose"][INIT_TICK + 1:] == 1).all(), tag      # every later tick yields a pose
    gt = lambda t: _gt(t, sc["speed"])
    ate, rot = isy.trajectory_errors(ticks, gt, t_align)
    G0 = np.linalg.inv(gt(t_align))
    still = float(np.sqrt(np.mean([np.sum((G0 @ gt(int(t)))[:3, 3] ** 2) for t in ticks[ticks["has_pose"] == 1]["t"]])))
    work = maps[maps["ran"] == 2]
    print(f"{tag}: ATE {ate * 1e3:.2f} mm (standing still: {still * 1e3:.1f} mm), max rotation error {rot:.3f} deg over "
          f"{int(ticks['has_pose'].sum())} poses; seeds per WORKING frame (median) {int(np.median(work['ctr'][:, 1]))}, "
          f"WORKING publishes {int(work['published'].sum())}, final map {m.size}")
    assert ate < sc["ate_m"] and ate < 0.6 * still and rot < sc["rot_deg"], (tag, ate, still, rot)
    if scene == "mapping":
        assert np.median(work["ctr"][:, 1]) >= 100, tag                                   # the denoised mapper solves seeds
        pub = work[work["published"] == 1]
        assert pub.size >= 3 and (pub["cloud_points"] >= 500).all(), tag                 # maps the tracker can adopt
        assert m.size >= 500, tag


@pytest.mark.parametrize("scene", list(SCENES))
def test_oracle_loop_tracks_ground_truth(oracle_lib, scene):
    """The restated loop on the oracle with the hkust yaml follows the ground truth."""
    import indep_system as isy
    s = _stream(scene)
    t0, n = _ticks(s)
    ticks, maps, m, traj, err = isy.run_system(_oracle(oracle_lib), _cv2_sgbm(), s["left"], s["right"], t0, DT_NS, n)
    assert err is None and ticks.size == n
    _check_follows_gt(ticks, maps, m, scene, f"oracle, {scene} scene")
    assert len(traj) == int(ticks["has_pose"].sum())


def test_oracle_reinitialises_when_map_is_too_small(oracle_lib):
    """BATCH_SIZE larger than any map: resetRegProblem fails at every pass (RegProblemSolverLM.cpp:52-57), the tracker sets
    INITIALIZATION again (esvo_Tracking.cpp:163-167) and the mapper re-runs the SGM start-up at every mapping tick."""
    import indep_system as isy
    s = _stream()
    t0, _ = _ticks(s)
    n = 40
    def tweak(p):
        p.trk_batch_size = HUGE_BATCH[1]
    ticks, maps, _, traj, err = isy.run_system(_oracle(oracle_lib, tweak), _cv2_sgbm(), s["left"], s["right"], t0, DT_NS, n)
    assert err is None and (ticks["status"] == 0).all() and (ticks["has_pose"] == 0).all() and not traj
    late = maps[maps["tick"] >= INIT_TICK]
    assert late.size == 6 and (late["ran"] == 1).all() and (late["ok"] == 1).all() and (late["published"] == 1).all()
    assert (maps[maps["tick"] < INIT_TICK]["ran"] == 0).all()


# ---------------------------------------------------------------- the example
def _build_example(exe):
    subprocess.check_call(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "system_loop.cpp"),
                           "-L" + BUILD, "-lesvo_b200", "-Wl,-rpath," + BUILD, "-o", exe])


def test_system_loop_builds_and_fails_cleanly_without_gpu(product_lib, tmp_path):
    import indep_system as isy
    exe = str(tmp_path / "system_loop")
    _build_example(exe)
    if has_gpu():
        return
    e = dict(x=np.zeros(1, np.uint16), y=np.zeros(1, np.uint16), t=np.ones(1, np.int64), p=np.zeros(1, np.uint8))
    isy.write_scenario(tmp_path / "s.bin", 346, 260, DT_NS, DT_NS, 3, e, e)
    p = subprocess.run([exe, str(tmp_path / "s.bin"), str(tmp_path / "r.bin"), str(tmp_path / "traj.txt")], capture_output=True, text=True)
    assert p.returncode == 2 and "no CPU fallback" in p.stdout, p.stdout + p.stderr


# ---------------------------------------------------------------- GPU: the same stream three ways
def _run_shim(tmp_path, s, t0, n, overrides=()):
    import indep_system as isy
    exe = str(tmp_path / "system_loop")
    _build_example(exe)
    scen, res, traj = tmp_path / "scen.bin", tmp_path / "res.bin", tmp_path / "traj.txt"
    isy.write_scenario(scen, 346, 260, t0, DT_NS, n, s["left"], s["right"], overrides=overrides)
    p = subprocess.run([exe, str(scen), str(res), str(traj)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    print(p.stdout.strip())
    return isy.parse_result(res), traj


def _first_difference(a_ticks, a_maps, b_ticks, b_maps, pose_tol, exact_counters):
    """The first tick and stage at which two runs differ, or None."""
    keys = ["ran", "ok", "published", "n_sgm_points", "cloud_points", "stamp"]
    mi = {int(m["tick"]): m for m in a_maps}; mj = {int(m["tick"]): m for m in b_maps}
    for k in range(max(a_ticks.size, b_ticks.size)):
        if k >= a_ticks.size or k >= b_ticks.size:
            return k, "run length"
        x, y = a_ticks[k], b_ticks[k]
        if x["t"] != y["t"] or x["status"] != y["status"] or x["has_pose"] != y["has_pose"]:
            return k, f"tracking: status {x['status']} / {y['status']}, pose {x['has_pose']} / {y['has_pose']}"
        d = np.abs(x["T"] - y["T"]).max()
        if (pose_tol == 0 and not np.array_equal(x["T"], y["T"])) or d > pose_tol:
            return k, f"tracking: pose differs by {d:.3g}"
        if (k in mi) != (k in mj):
            return k, "mapping: ran on one side only"
        if k in mi:
            u, v = mi[k], mj[k]
            for key in keys:
                if u[key] != v[key]:
                    return k, f"mapping: {key} {u[key]} / {v[key]}"
            cu, cv = u["ctr"], v["ctr"]
            idx = range(8) if exact_counters else (0, 1, 2, 3, 4, 7)   # bm_evals / lm_evals are work counters
            for i in idx:
                if cu[i] != cv[i]:
                    import indep_system as isy
                    return k, f"mapping: {isy.CTR_KEYS[i]} {cu[i]} / {cv[i]}"
    return None


@pytest.mark.gpu
@pytest.mark.parametrize("scene", list(SCENES))
def test_system_loop_same_stream_three_ways(oracle_lib, product_lib, tmp_path, scene):
    """Shim and restatement on the product give identical outputs; product and oracle meet the parity bar of
    test_shim_mapping_to_tracking_matches_oracle at every tick and for the final map; the trajectory file parses back to the
    returned poses."""
    import indep_system as isy
    from util import make_backends
    s = _stream(scene)
    t0, n = _ticks(s)
    (sh_ticks, sh_maps, sh_map, stopped, wall, _, _), traj = _run_shim(tmp_path, s, t0, n)
    assert stopped == 0 and sh_ticks.size == n
    o, g = make_backends("hkust", oracle_lib, product_lib)
    pr_ticks, pr_maps, pr_map, _, err = isy.run_system(g, lambda l, r: g.sgbm_compute(l, r), s["left"], s["right"], t0, DT_NS, n)
    assert err is None
    # 1. shim vs restatement, both on the product: identical
    diff = _first_difference(sh_ticks, sh_maps, pr_ticks, pr_maps, 0.0, True)
    assert diff is None, f"shim vs restatement on the product: first difference at tick {diff[0]}: {diff[1]}"
    assert sh_map.tobytes() == pr_map.tobytes()
    # 2. product vs oracle, tick by tick, and the final map
    or_ticks, or_maps, or_map, _, err = isy.run_system(o, _cv2_sgbm(), s["left"], s["right"], t0, DT_NS, n)
    assert err is None
    pose_err = np.abs(pr_ticks["T"] - or_ticks["T"]).max()
    print(f"product vs oracle: largest pose difference {pose_err:.3g} over {n} ticks; shim loop {wall:.0f} ms")
    diff = _first_difference(pr_ticks, pr_maps, or_ticks, or_maps, 1e-6, False)
    assert diff is None, f"product vs oracle: first difference at tick {diff[0]}: {diff[1]}"
    assert pr_map.size == or_map.size
    assert np.array_equal(pr_map["row"], or_map["row"]) and np.array_equal(pr_map["col"], or_map["col"])
    if scene == "mapping":
        rel = np.abs(pr_map["inv_depth"] - or_map["inv_depth"]) / np.abs(or_map["inv_depth"])
        assert pr_map.size >= 500 and (rel < 1e-4).mean() >= 0.999, (pr_map.size, rel.max())
    # 3. the bounds hold on the product; the trajectory file parses back to the returned poses
    _check_follows_gt(sh_ticks, sh_maps, sh_map, scene, f"product, {scene} scene")
    from scipy.spatial.transform import Rotation
    st, rows = isy.read_trajectory(traj)
    posed = sh_ticks[sh_ticks["has_pose"] == 1]
    assert st.size == posed.size and np.abs(st - posed["t"] * 1e-9).max() < 1e-6
    for row, r in zip(rows, posed):
        T = r["T"].reshape(4, 4)
        q = Rotation.from_matrix(T[:3, :3]).as_quat()
        assert np.abs(row[:3] - T[:3, 3]).max() < 1e-9
        assert min(np.abs(row[3:] - q).max(), np.abs(row[3:] + q).max()) < 1e-9


@pytest.mark.gpu
def test_system_loop_reinitialisation_matches_oracle(oracle_lib, product_lib, tmp_path):
    """BATCH_SIZE larger than any map on the GPU: the shim re-initialises at every mapping tick like the oracle, tick by tick."""
    import indep_system as isy
    from util import make_backends
    s = _stream()
    t0, _ = _ticks(s)
    n = 40
    (sh_ticks, sh_maps, _, stopped, _, _, _), _ = _run_shim(tmp_path, s, t0, n, (HUGE_BATCH,))
    def tweak(p):
        p.trk_batch_size = HUGE_BATCH[1]
    o, g = make_backends("hkust", oracle_lib, product_lib, tweak)
    g.close()
    or_ticks, or_maps, _, _, err = isy.run_system(o, _cv2_sgbm(), s["left"], s["right"], t0, DT_NS, n)
    assert stopped == 0 and err is None
    diff = _first_difference(sh_ticks, sh_maps, or_ticks, or_maps, 0.0, False)
    assert diff is None, f"first difference at tick {diff[0]}: {diff[1]}"
    assert (sh_ticks["status"] == 0).all() and (sh_maps[sh_maps["tick"] >= INIT_TICK]["ran"] == 1).all()
