"""Fusion-stage timing probe at pipeline depth 1: the bench frame's fusion (stage + order + fold + regularise + commit) alone,
CUDA events of the library's profile stage 5.  usage: python scripts/fold_probe.py [cfg2|cfg3]"""
import ctypes as C, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from esvo_b200 import capi, configs
cfgname = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
cfg = bench.CONFIGS[cfgname]
prod = capi.load_product()
l, r = configs.rig_calibs(cfg["rig"])
prm = configs.params_for(cfg["rig"], prod)
g = capi.Backend(prod, l, r, prm)
base = bench.make_workload(seed=10 if cfgname == "cfg2" else 3, cfg=cfgname)
f64, u64 = C.POINTER(C.c_double), C.POINTER(C.c_uint64)
n_prime = prm.max_num_fusion_frames
ts = []
for k in range(n_prime + 6):
    f = bench.shifted(base, k)
    for cam, side in ((0, "left"), (1, "right")):
        e = f[side]; g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"]); g.ts_build(cam, f["t_ts_ns"], want_idx=False, want_ts=False)
    g.set_ts_pair(None, None, f["T_world_left"])
    sd = f["seeds"]
    if k >= n_prime:
        g._call("profile", [C.c_int], 0xFF); g._call("profile_read", [f64, u64], (C.c_double * 8)(), (C.c_uint64 * 8)())
    c = g.mapping_at_time(sd["x"], sd["y"], sd["t"], f["pose_t"], f["poses"])
    if k >= n_prime:
        ms = (C.c_double * 8)(); cnt = (C.c_uint64 * 8)()
        g._call("profile_read", [f64, u64], ms, cnt); g._call("profile", [C.c_int], 0)
        ts.append(list(ms)[:6])
ts = np.array(ts)
print(cfgname, "stage ms [ts, bm, seed order, lm, point order, fusion]:", np.round(np.median(ts, axis=0), 4).tolist(), "n_fusions", c["n_fusions"], "map", c["map_size"])
