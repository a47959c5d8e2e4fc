"""Measures the closed loop fed from a ROS bag (examples/bag_system.cpp: events copied as wire records out of the mapped bag,
decoded on the device) against the same loop fed SoA vectors (examples/system_loop.cpp), on the same seeded hkust scenes
(tests/test_system_loop.py's), and an isolated packed push against the SoA push.  Prints one JSON line: the card and its
power limit; per scene and runner (alternating, --runs each) the wall time per second of stream and the host ms per tick of
ts.eventsCallback; and the median of --reps pushes of 64 Ki and 1 Mi events, host call to device completion (CUDA-event
timed on the context's stream is not reachable from Python; the push is followed by esvo_sync), for
esvo_ts_push_events, esvo_ts_push_event_array and esvo_ts_push_event_array_dev.
Builds the examples and writes the scenario and bag files into a temporary directory; writes nothing in the tree.
usage: python scripts/bag_probe.py [--seconds 2.0] [--seed 2] [--runs 3] [--reps 20]"""
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
SCENES = {"dense": dict(), "mapping": dict(n_segments=7, speed=2.0, depth_range=(0.5, 1.2))}
L, R, LI, RI = "/davis/left/events", "/davis/right/events", "/davis/left/camera_info", "/davis/right/camera_info"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def compile_example(tmp, name):
    build = os.path.join(ROOT, "esvo_b200", "_build")
    exe = os.path.join(tmp, name)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", name + ".cpp"),
                           "-L" + build, "-lesvo_b200", "-Wl,-rpath," + build, "-o", exe])
    return exe


def run(cmd, tmp, seconds):
    import indep_system as isy
    calls = os.path.join(tmp, "calls.txt")
    p = subprocess.run(cmd(calls), capture_output=True, text=True)
    if p.returncode:
        raise SystemExit(p.stdout + p.stderr)
    ticks, _, _, _, wall, _, _ = isy.parse_result(os.path.join(tmp, "r.bin"))
    ev = [ln.split() for ln in open(calls) if ln.startswith("ts.eventsCallback ")][0]
    return wall / seconds, float(ev[1]) / max(int(ev[2]), 1)


def loop(a, tmp):
    import indep_system as isy
    import rosbag_writer as rw
    from esvo_b200 import configs, synth
    sl, bs = compile_example(tmp, "system_loop"), compile_example(tmp, "bag_system")
    rr = configs.RIGS["hkust"]
    infos = {t: (rr["width"], rr["height"], rr["model"], rr[sd]["D"], rr[sd]["K"], rr[sd]["R"], rr[sd]["P"]) for t, sd in ((LI, "left"), (RI, "right"))}
    out = {}
    for scene, kw in SCENES.items():
        s = synth.make_stream("hkust", seed=a.seed, t_ts=a.seconds, history_ms=a.seconds * 1e3, **kw)
        t0 = s["t_ts_ns"] - int(round(a.seconds * 1e9)) + DT_NS
        n = int(round(a.seconds * 1e9 / DT_NS))
        scen, bag = os.path.join(tmp, "s.bin"), os.path.join(tmp, "s.bag")
        isy.write_scenario(scen, 346, 260, t0, DT_NS, n, s["left"], s["right"])
        rw.write_event_bag(bag, {L: s["left"], R: s["right"]}, infos=infos, msg_events=1500, chunk_threshold=768 * 1024)
        res, traj = os.path.join(tmp, "r.bin"), os.path.join(tmp, "t.txt")
        cmds = {"system_loop": lambda c: [sl, scen, res, traj, c],
                "bag_system": lambda c: [bs, bag, L, R, LI, RI, res, traj, "--t0-ns", str(t0), "--dt-ns", str(DT_NS), "--ticks", str(n), "--calls", c]}
        got = {k: ([], []) for k in cmds}
        for _ in range(a.runs):
            for k, cmd in cmds.items():
                w, e = run(cmd, tmp, a.seconds)
                got[k][0].append(round(w, 1)); got[k][1].append(round(e, 4))
        out[scene] = {k: {"wall_ms_per_stream_s": v[0], "ts_eventsCallback_host_ms_per_tick": v[1]} for k, v in got.items()}
    return out


def pushes(a):
    import torch
    from esvo_b200 import capi, configs
    lib = capi.load_product()
    l, r = configs.rig_calibs("hkust")
    b = capi.Backend(lib, l, r, configs.params_for("hkust", lib))
    out = {}
    for n in (1 << 16, 1 << 20):
        rng = np.random.default_rng(n)
        t = (1_600_000_000 * 10**9 + np.cumsum(rng.integers(0, 100, n * (a.reps + 2)))).astype(np.int64)
        x = rng.integers(0, 346, t.size).astype(np.uint16); y = rng.integers(0, 260, t.size).astype(np.uint16)
        p = rng.integers(0, 2, t.size).astype(np.uint8)
        rec = capi.pack_events(x, y, t, p)
        dev = torch.from_numpy(rec.view(np.uint8).copy()).cuda()
        res = {}
        for name in ("soa", "packed_host", "packed_dev"):
            b.ts_reset(0)
            ms = []
            for k in range(a.reps + 2):
                sl = slice(k * n, (k + 1) * n)
                c0 = time.perf_counter()
                if name == "soa":
                    b.ts_push_events(0, x[sl], y[sl], t[sl], p[sl])
                elif name == "packed_host":
                    b.ts_push_event_array(0, [rec[sl].view(np.uint8)])
                else:
                    b.ts_push_event_array_dev(0, dev.data_ptr() + 13 * k * n, n)
                b._call("sync", [])
                ms.append((time.perf_counter() - c0) * 1e3)
            res[name] = round(float(np.median(ms[2:])), 4)
        out[f"{n}_events_ms"] = res
    b.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    out = {"workload": f"hkust synthetic scenes, seed {a.seed}, {a.seconds:g} s at 100 Hz ticks, hkust yaml; bag: 1 500 events per "
                       "EventArray, 768 KiB chunks, Imu and Image topics interleaved"}
    out["gpu"], out["power_limit"] = card()
    with tempfile.TemporaryDirectory() as tmp:
        out["loop"] = loop(a, tmp)
    out["push"] = pushes(a)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
