"""Measures the closed loop (examples/system_loop.cpp, esvo_core::esvo_System) on a seeded 2 s hkust stream and prints one
JSON line: the card and its power limit, wall time per second of stream, mapping / tracking / time-surface ms, the per-stage
esvo_profile breakdown, the host time of every call SpinOnce and MappingLoopOnce make (ms per tick or per mapping frame that
made the call), when tracking starts, how well it follows the ground truth, and the same stream through the Python
restatement (tests/indep_system.py) on the CPU oracle.  Scenes as in tests/test_system_loop.py: "dense" (the default
80-segment scene) and "mapping" (7 segments at 0.5-1.2 m, twice the speed: WORKING maps are published and adopted).
--root: the tree whose library and example are measured (default: this one), to compare builds in one session.
Builds the example into a temporary directory; writes nothing in the tree.
usage: python scripts/loop_probe.py [--seconds 2.0] [--seed 2] [--scene dense|mapping] [--root DIR] [--no-oracle]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
DT_NS = 10_000_000
SCENES = {"dense": (dict(), 1.0), "mapping": (dict(n_segments=7, speed=2.0, depth_range=(0.5, 1.2)), 2.0)}
STAGES = ["time_surface", "block_matching", "seed_ordering", "depth_lm", "point_ordering_culling", "fusion_clean_regularise", "tracking", "stage7"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--scene", choices=list(SCENES), default="dense")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import indep_system as isy
    from esvo_b200 import synth
    kw, speed = SCENES[a.scene]
    s = synth.make_stream("hkust", seed=a.seed, t_ts=a.seconds, history_ms=a.seconds * 1e3, **kw)
    t0 = s["t_ts_ns"] - int(round(a.seconds * 1e9)) + DT_NS
    n = int(round(a.seconds * 1e9 / DT_NS))
    gt = lambda t: synth.pose_at(t * 1e-9 * speed)
    out = {"workload": f"hkust synthetic stream, {a.scene} scene, seed {a.seed}, {a.seconds:g} s, {n} ticks at 100 Hz, mapping at 20 Hz, "
                       f"hkust yaml", "root": os.path.abspath(a.root)}
    out["gpu"], out["power_limit"] = card()
    with tempfile.TemporaryDirectory() as tmp:
        build = os.path.join(a.root, "esvo_b200", "_build")
        exe = os.path.join(tmp, "system_loop")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(a.root, "include"), os.path.join(a.root, "examples", "system_loop.cpp"),
                               "-L" + build, "-lesvo_b200", "-Wl,-rpath," + build, "-o", exe])
        isy.write_scenario(os.path.join(tmp, "s.bin"), 346, 260, t0, DT_NS, n, s["left"], s["right"], profile=True)
        calls_path = os.path.join(tmp, "calls.txt")
        p = subprocess.run([exe, os.path.join(tmp, "s.bin"), os.path.join(tmp, "r.bin"), os.path.join(tmp, "t.txt"), calls_path],
                           capture_output=True, text=True)
        if p.returncode:
            raise SystemExit(p.stdout + p.stderr)
        ticks, maps, m, stopped, wall, prof_ms, prof_n = isy.parse_result(os.path.join(tmp, "r.bin"))
        calls = {}
        if os.path.exists(calls_path):            # a tree whose example writes no call times has no breakdown
            for line in open(calls_path):
                name, total, count = line.split()
                calls[name] = {"ms_per_call": round(float(total) / max(int(count), 1), 4), "calls": int(count)}
    ms = ticks["ms"]
    mapped = np.isin(np.arange(ticks.size), maps[maps["ran"] == 2]["tick"])
    posed = ticks["has_pose"] == 1
    q = lambda v, p: round(float(np.percentile(v, p)), 3) if v.size else None
    out["wall_ms_per_stream_s"] = round(wall / a.seconds, 1)
    out["mapping_ms_per_frame"] = {"median": q(ms[mapped, 2], 50), "p90": q(ms[mapped, 2], 90), "frames": int(mapped.sum())}
    out["init_ms"] = [round(float(ms[int(k), 2]), 3) for k in maps[maps["ran"] == 1]["tick"]]
    out["tracking_ms_per_frame"] = {"median": q(ms[posed, 1], 50), "p90": q(ms[posed, 1], 90)}
    out["ts_ms_per_tick"] = {"median": q(ms[:, 0], 50), "p90": q(ms[:, 0], 90)}
    out["profile_ms"] = {STAGES[i]: round(float(prof_ms[i]), 3) for i in range(8) if prof_n[i]}
    out["profile_launches"] = {STAGES[i]: int(prof_n[i]) for i in range(8) if prof_n[i]}
    out["host_ms_per_call"] = calls
    out["first_pose_tick"] = int(np.argmax(posed)) if posed.any() else None
    out["tracked_frames"] = int(posed.sum())
    out["stopped"] = bool(stopped)
    t_align = int(maps[(maps["ran"] == 1) & (maps["ok"] == 1)][0]["stamp"])
    ate, rot = isy.trajectory_errors(ticks, gt, t_align)
    out["ate_m"], out["max_rot_err_deg"] = round(ate, 5), round(rot, 3)
    out["final_map_points"] = int(m.size)
    if not a.no_oracle:
        import cv2
        from esvo_b200 import capi, configs
        from oracle.loader import load_oracle
        orc = load_oracle()
        l, r = configs.rig_calibs("hkust")
        o = capi.Backend(orc, l, r, configs.params_for("hkust", orc))
        sg = cv2.StereoSGBM_create(0, 48, 11, 968, 3872, -1, 0, 11)
        c0 = time.perf_counter()
        ot, om, _, _, err = isy.run_system(o, lambda x, y: sg.compute(x, y), s["left"], s["right"], t0, DT_NS, n)
        wall_o = (time.perf_counter() - c0) * 1e3
        ate_o, rot_o = isy.trajectory_errors(ot, gt, int(om[(om["ran"] == 1) & (om["ok"] == 1)][0]["stamp"]))
        out["oracle_restatement"] = {"host_cores": os.cpu_count(), "wall_ms_per_stream_s": round(wall_o / a.seconds, 1),
                                     "tracked_frames": int(ot["has_pose"].sum()), "ate_m": round(ate_o, 5), "max_rot_err_deg": round(rot_o, 3),
                                     "error": err}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
