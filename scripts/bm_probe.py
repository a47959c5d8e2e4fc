"""BM kernel probe: esvo_bm_match on the bench workloads (hkust 5k events, dsec 20k events); prints the isolated kernel time
(esvo_profile stage 1) and a digest of the seeds so that two builds can be compared."""
import ctypes as C, hashlib, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from esvo_b200 import capi, configs, synth
prod = capi.load_product()
f64, u64 = C.POINTER(C.c_double), C.POINTER(C.c_uint64)
for rig, n, kw in (("hkust", 5000, {}), ("dsec", 20000, dict(n_segments=120))):
    s = synth.make_stream(rig, seed=10 if rig == "hkust" else 3, n_seeds=n, history_ms=50.0, **kw)
    l, r = configs.rig_calibs(rig)
    g = capi.Backend(prod, l, r, configs.params_for(rig, prod))
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]; g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"]); g.ts_build(cam, s["t_ts_ns"], want_idx=False, want_ts=False)
    g.set_ts_pair(None, None, s["T_world_left"])
    g._call("profile", [C.c_int], 1 << 1)
    sd = s["seeds"]
    ts = []
    for _ in range(5):
        seeds, ev = g.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        m, c = (C.c_double * 8)(), (C.c_uint64 * 8)()
        g._call("profile_read", [f64, u64], m, c)
        ts.append(m[1])
    print(f"{rig}: bm kernel {min(ts[1:]) * 1e3:.1f} us, seeds {seeds.size}, evals {ev}, digest {hashlib.md5(seeds.tobytes()).hexdigest()[:12]}")
    g.close()
