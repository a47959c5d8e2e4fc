"""Measures hot-pixel removal (include/esvo_b200_hotpix.h).  Prints one JSON line with the card and its power limit and:
  * count: esvo_hotpix_count_event_array_dev over --dev-events wire records in device memory, and esvo_hotpix_count_event_array
    over --host-events records in host runs of 1 500 (one EventArray each), in events per second (host clock around the call
    and esvo_sync, median of --reps);
  * loop: examples/bag_system.cpp on the hkust scenes of tests/test_system_loop.py (seed 2) with 20 hot pixels per camera
    injected as tests/test_gpu_hot_pixels.py does, without and with --hot-pixels 5 (alternating, --runs each): wall ms per
    second of stream (the loop only, after the count and selection), and how far the unfiltered trajectory lies from the
    filtered one (translation RMS / max in mm, rotation max in degrees, over the ticks where both have a pose).
Builds bag_system and writes the bags into a temporary directory; writes nothing in the tree.
usage: python scripts/hotpix_probe.py [--runs 2] [--reps 3] [--dev-events 200000000] [--host-events 20000000]"""
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bag_probe import DT_NS, L, LI, R, RI, card, compile_example  # noqa: E402


def counting(a):
    import torch
    from esvo_b200 import capi, configs
    lib = capi.load_product()
    l, r = configs.rig_calibs("hkust")
    b = capi.Backend(lib, l, r, configs.params_for("hkust", lib))
    rng = np.random.default_rng(3)
    n = a.host_events
    rec = capi.pack_events(rng.integers(0, 346, n), rng.integers(0, 260, n), 1_600_000_000 * 10**9 + np.arange(n), rng.integers(0, 2, n))
    hot = rng.random(n) < 0.05
    rec["x"][hot] = rng.integers(0, 20, int(hot.sum())) * 17
    raw = rec.view(np.uint8)
    runs = [raw[13 * k:13 * min(n, k + 1500)] for k in range(0, n, 1500)]
    dev = torch.from_numpy(raw.copy()).cuda().repeat((a.dev_events + n - 1) // n)[:13 * a.dev_events]
    torch.cuda.synchronize()
    out = {}
    for name, call in (("dev", lambda: b.hotpix_count_event_array_dev(0, dev.data_ptr(), a.dev_events)),
                       ("host_runs_of_1500", lambda: b.hotpix_count_event_array(0, runs))):
        events = a.dev_events if name == "dev" else n
        s = []
        for _ in range(a.reps + 1):
            b.hotpix_clear(0); b._call("sync", [])
            c0 = time.perf_counter()
            call(); b._call("sync", [])
            s.append(time.perf_counter() - c0)
        out[f"{name}_events_per_s"] = round(events / float(np.median(s[1:])), -6)
        out[f"{name}_events"] = events
    b.close()
    return out


def pose_gap(a_ticks, b_ticks):
    from scipy.spatial.transform import Rotation
    both = (a_ticks["has_pose"] == 1) & (b_ticks["has_pose"] == 1)
    A, B = a_ticks["T"][both].reshape(-1, 4, 4), b_ticks["T"][both].reshape(-1, 4, 4)
    d = np.linalg.norm(A[:, :3, 3] - B[:, :3, 3], axis=1)
    rot = Rotation.from_matrix(np.einsum("nji,njk->nik", A[:, :3, :3], B[:, :3, :3])).magnitude()
    return {"poses": int(both.sum()), "trans_rms_mm": round(float(np.sqrt(np.mean(d ** 2))) * 1e3, 3),
            "trans_max_mm": round(float(d.max()) * 1e3, 3), "rot_max_deg": round(float(np.degrees(rot.max())), 4)}


def loop(a, tmp):
    import indep_system as isy
    import rosbag_writer as rw
    import test_gpu_hot_pixels as thp
    import test_system_loop as tsl
    from esvo_b200 import configs
    bs = compile_example(tmp, "bag_system")
    rr = configs.RIGS["hkust"]
    infos = {t: (rr["width"], rr["height"], rr["model"], rr[sd]["D"], rr[sd]["K"], rr[sd]["R"], rr[sd]["P"]) for t, sd in ((LI, "left"), (RI, "right"))}
    out = {}
    for scene in ("dense", "mapping"):
        s = tsl._stream(scene)
        t0, n = tsl._ticks(s)
        pix = np.random.default_rng(62).choice(346 * 260, 2 * thp.N_HOT, replace=False)
        bag = os.path.join(tmp, "s.bag")
        rw.write_event_bag(bag, {L: thp._inject(s["left"], pix[:thp.N_HOT], 346, 63), R: thp._inject(s["right"], pix[thp.N_HOT:], 346, 64)},
                           infos=infos, msg_events=1500, chunk_threshold=768 * 1024)
        res, traj = os.path.join(tmp, "r.bin"), os.path.join(tmp, "t.txt")
        got, ticks = {"unfiltered": [], "hot_pixels_5": []}, {}
        for _ in range(a.runs):
            for k in got:
                cmd = [bs, bag, L, R, LI, RI, res, traj, "--t0-ns", str(t0), "--dt-ns", str(DT_NS), "--ticks", str(n)]
                p = subprocess.run(cmd + (["--hot-pixels", "5"] if k != "unfiltered" else []), capture_output=True, text=True)
                if p.returncode:
                    raise SystemExit(p.stdout + p.stderr)
                r = isy.parse_result(res)
                got[k].append(round(r[4] / tsl.DURATION_S, 1))
                ticks[k] = r[0]
        out[scene] = {"wall_ms_per_stream_s": got, "unfiltered_vs_filtered": pose_gap(ticks["unfiltered"], ticks["hot_pixels_5"])}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dev-events", type=int, default=200_000_000)
    ap.add_argument("--host-events", type=int, default=20_000_000)
    a = ap.parse_args()
    out = {"workload": "count: 5 % of the records on 20 pixels; loop: hkust scenes, seed 2, 1.3 s at 100 Hz ticks, 20 hot pixels "
                       "per camera at 500 Hz - 5 kHz, bag of 1 500 events per EventArray"}
    out["gpu"], out["power_limit"] = card()
    out["count"] = counting(a)
    with tempfile.TemporaryDirectory() as tmp:
        out["loop"] = loop(a, tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
