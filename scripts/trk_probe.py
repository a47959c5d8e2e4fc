"""Tracking solver timing probe: reset + solve on the bench workload's fused map (host wall clock around the synchronous calls)."""
import os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from esvo_b200 import capi, configs, synth
prod = capi.load_product()
s = synth.make_stream("hkust", seed=10, n_seeds=5000, history_ms=50.0)
s2 = synth.make_stream("hkust", seed=10, n_seeds=100, history_ms=50.0, t_ts=0.51)
l, r = configs.rig_calibs("hkust")
g = capi.Backend(prod, l, r, configs.params_for("hkust", prod))
for cam, side in ((0, "left"), (1, "right")):
    e = s[side]; g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"]); g.ts_build(cam, s["t_ts_ns"], want_idx=False, want_ts=False)
g.set_ts_pair(None, None, s["T_world_left"])
sd = s["seeds"]
g.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
m = g.map_download()
Tw = np.asarray(s["T_world_left"], float)
cloud = (m["p_cam"] @ Tw[:3, :3].T + Tw[:3, 3]).astype(np.float32)
g.ts_reset(0); e = s2["left"]; g.ts_push_events(0, e["x"], e["y"], e["t"], e["p"])
_, ts_cur = g.ts_build(0, s2["t_ts_ns"], want_idx=False)
for analytical in (True, False):
    tt = []
    for rep in range(10):
        c = cloud.copy(); g.track_srand(1)
        t0 = time.perf_counter(); g.track_reset(c, Tw, Tw, ts_cur); t1 = time.perf_counter(); T, st = g.track_solve(analytical); t2 = time.perf_counter()
        tt.append(((t1 - t0) * 1e3, (t2 - t1) * 1e3))
    tt = np.array(tt[2:])
    print(f"analytical={analytical}: reset {np.median(tt[:,0]):.3f} ms solve {np.median(tt[:,1]):.3f} ms stats {st} pose t {T[:3,3]}")
