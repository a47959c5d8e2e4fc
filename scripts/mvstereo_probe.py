"""Measures the multi-view stereo system (examples/mvstereo_system.cpp, esvo_core::esvo_MVStereoSystem) in each of its five
modes on a seeded 2 s synthetic stream with its ground-truth pose stream, esvo_profile on, and prints one JSON line: the
card and its power limit, and per mode the wall time per second of stream, the mapping ms per frame and the per-stage
device time.  Builds the example into a temporary directory; writes nothing in the tree.
usage: python scripts/mvstereo_probe.py [--rig rpg|upenn] [--seconds 2.0] [--seed 3]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
DT_NS = 10_000_000
STAGES = ["time_surface", "block_matching", "seed_ordering", "depth_lm", "point_ordering_culling", "fusion_clean_regularise", "tracking", "stage7"]
MODES = ["PURE_EVENT_MATCHING", "PURE_BLOCK_MATCHING", "EM_PLUS_ESTIMATION", "BM_PLUS_ESTIMATION", "PURE_SEMI_GLOBAL_MATCHING"]
DEPTHS = {"rpg": (0.8, 3.0), "upenn": (1.2, 4.0)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rig", default="rpg", choices=sorted(DEPTHS))
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--seed", type=int, default=3)
    a = ap.parse_args()
    import indep_mvstereo as imv
    from esvo_b200 import capi, configs, synth
    lib = capi.load_product()
    s = synth.make_stream(a.rig, seed=a.seed, t_ts=a.seconds + 0.05, history_ms=(a.seconds + 0.05) * 1e3, n_seeds=10, n_segments=40,
                          depth_range=DEPTHS[a.rig], translation_scale=1.0, rig_model=True)
    pose_t = np.arange(int(s["left"]["t"][0]), s["t_ts_ns"] + 1, 1_000_000, dtype=np.int64)
    M = np.linalg.inv(imv.T_MARKER_CAM) if configs.mvstereo_config(a.rig)["dvs_frame_id"] == "marker" else np.eye(4)
    poses = np.array([(synth.pose_at(v * 1e-9) @ M).ravel() for v in pose_t])
    t0 = s["t_ts_ns"] - int(round(a.seconds * 1e9)) + DT_NS
    n = int(round(a.seconds * 1e9 / DT_NS))
    out = {"workload": f"{a.rig} synthetic stream, seed {a.seed}, {a.seconds:g} s, {s['left']['t'].size + s['right']['t'].size} events, "
                       f"{n} ticks at 100 Hz, mapping at 20 Hz, 1 kHz pose stream, mvstereo_{a.rig}.yaml"}
    out["gpu"], out["power_limit"] = card()
    l, r = configs.rig_calibs(a.rig)
    with tempfile.TemporaryDirectory() as tmp:
        build = os.path.join(ROOT, "esvo_b200", "_build")
        exe = os.path.join(tmp, "mvstereo_system")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "mvstereo_system.cpp"),
                               "-L" + build, "-lesvo_b200", "-Wl,-rpath," + build, "-o", exe])
        for mode, name in enumerate(MODES):
            cfg = dict(configs.mvstereo_config(a.rig), MVStereoMode=mode)
            scen, res = os.path.join(tmp, "s.bin"), os.path.join(tmp, "r.bin")
            imv.write_scenario(scen, l, r, configs.mvstereo_params_for(a.rig, lib), t0, DT_NS, n, cfg, s["left"], s["right"], pose_t, poses,
                               profile=True)
            p = subprocess.run([exe, scen, res], capture_output=True, text=True)
            if p.returncode:
                raise SystemExit(p.stdout + p.stderr)
            fr, m, stopped, wall, prof_ms, prof_n = imv.parse_result(res)
            ran = fr[fr["ran"] == 1]
            q = lambda v, pc: round(float(np.percentile(v, pc)), 3) if v.size else None
            out[name] = {"wall_ms_per_stream_s": round(wall / a.seconds, 1),
                         "mapping_ms_per_frame": {"median": q(ran["ms"], 50), "p90": q(ran["ms"], 90), "frames": int(ran.size)},
                         "profile_ms": {STAGES[i]: round(float(prof_ms[i]), 3) for i in range(8) if prof_n[i]},
                         "published": int(fr["published"].sum()), "final_map_points": int(m.size), "stopped": bool(stopped)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
