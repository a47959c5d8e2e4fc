"""Where the depth LM of the device and of the oracle part, off the shipped 15 x 7 shape (DESIGN.md section 9, LM tail).

The seeds of the default 15 x 7 block matching (the seeds of tests/test_gpu_parity.py::test_depth_solver_parity) are solved by
both sides at max_iteration K = 1 .. 10.  For every seed whose inverse depth ends more than 1e-7 apart, the first K at which
rho, the variance or the cost part is classified from the oracle's iterates (esvo_oracle_op_depth_solve_trace) with the
restatement of tests/indep_numpy.py, at the last agreed iterate, the two parted iterates and their forward-difference points:
  failed-warp  the warp fails at some of these points and not at others;
  stall        the scale iteration ends at a subnormal scale (|f| < 1e-100) at some of them;
  rounding-5%  a 5 % test of the scale iteration is decided within 1e-9 of its threshold;
  lmpar        none of these: the step itself differs.
Also scans util.DEPTH_CASES at K = 1 .. 10.  Needs a GPU.  Usage: python scripts/lm_tail_probe.py OUT.json
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import indep_numpy as ind  # noqa: E402
from esvo_b200 import capi, configs  # noqa: E402
from oracle.loader import load_oracle  # noqa: E402
from util import DEPTH_CASES, build_ts_pair, depth_inputs, depth_params, make_backends, scenario  # noqa: E402

HEPS = 1.4901161193847656e-08
SHAPES = [(1, 1), (3, 3), (15, 1), (1, 15), (5, 5), (17, 5), (7, 15), (37, 3), (113, 1), (23, 5), (13, 9), (17, 7), (11, 11), (127, 1)]


def rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


def solve_map(be, seeds):
    pts, _ = be.depth_solve(seeds)
    return {(float(p["x"][0]), float(p["x"][1])): (float(p["inv_depth"]), float(p["variance"]), float(p["residual"])) for p in pts}


def classify(o, seed, Tlw, Pl, Pr, tl, tr, wx, wy, p, xs):
    T = Tlw @ seed["T_world_virtual"].reshape(4, 4)
    failed, stall, margin = [], False, np.inf
    for x in xs:
        for xx in (x, x + HEPS * abs(x)):
            info = {}
            f = ind.depth_residual(xx, seed["x_left"], T, Pl, Pr, tl, tr, wx, wy, p.td_nu, p.td_scale, "Tdist", info)
            failed.append(info["failed"])
            if not info["failed"]:
                stall |= bool(np.abs(f).max() < 1e-100)
                margin = min(margin, info["margin"])
    if any(failed) and not all(failed):
        return "failed-warp"
    if stall:
        return "stall"
    if margin < 1e-9:
        return "rounding-5%"
    return "lmpar"


def main(out):
    prod, orc = capi.load_product(), load_oracle()
    orc.lib.esvo_oracle_set_irls_shortcut(1)     # outcome-identical to the literal loop under the guard (DESIGN.md deviation 4)
    trace_fn = orc.lib.esvo_oracle_op_depth_solve_trace
    trace_fn.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.c_int]
    trace_fn.restype = C.c_int
    res = dict(tail={}, cases={})
    s = scenario("hkust")
    o0, g0 = make_backends("hkust", orc, prod)
    tl, tr = build_ts_pair(o0, s)
    o0.set_ts_pair(tl, tr, s["T_world_left"])
    sd = s["seeds"]
    seeds, _ = o0.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    A = configs.rig_arrays("hkust")
    Pl, Pr = A["left"]["P"], A["right"]["P"]
    Tlw = np.linalg.inv(s["T_world_left"])
    key = {(float(q["x_left"][0]), float(q["x_left"][1])): i for i, q in enumerate(seeds)}
    for wx, wy in SHAPES:
        per_k = []
        for K in range(1, 11):
            def tw(p, K=K):
                p.patch_size_x, p.patch_size_y, p.max_iteration = wx, wy, K
            o, g = make_backends("hkust", orc, prod, tweak=tw)
            for be in (o, g):
                be.set_ts_pair(tl, tr, s["T_world_left"])
            per_k.append((solve_map(o, seeds), solve_map(g, seeds), o))
        mo, mg, o10 = per_k[-1]
        parted = [k for k in mo if k in mg and rel(mg[k][0], mo[k][0]) > 1e-7]
        rows = []
        for k in parted:
            first = next((K for K in range(1, 11) if k in per_k[K - 1][0] and k in per_k[K - 1][1] and
                          (rel(per_k[K - 1][1][k][0], per_k[K - 1][0][k][0]) > 1e-9 or
                           rel(per_k[K - 1][1][k][1], per_k[K - 1][0][k][1]) > 1e-6 or
                           rel(per_k[K - 1][1][k][2], per_k[K - 1][0][k][2]) > 1e-6)), None)
            seed = seeds[key[k]]
            tb = np.zeros(40)
            n = trace_fn(o10.ctx, np.ascontiguousarray(seed.reshape(1)).ctypes.data_as(C.c_void_p), tb.ctypes.data_as(C.POINTER(C.c_double)), 20)
            xo = [float(seed["inv_depth"])] + [tb[2 * i] for i in range(max(n, 0))]
            K = first or 10
            pts = [xo[min(K - 1, len(xo) - 1)], xo[min(K, len(xo) - 1)], per_k[K - 1][1][k][0]]
            cls = classify(o10, seed, Tlw, Pl, Pr, tl, tr, wx, wy, o10.params, pts)
            rows.append(dict(x=k, first_K=first, cls=cls, rho_o=mo[k][0], rho_g=mg[k][0], cost_o=mo[k][2]))
        res["tail"][f"{wx}x{wy}"] = dict(n=len(mo), parted=rows)
        print(f"{wx}x{wy}: {len(mo)} solved, {len(parted)} parted beyond 1e-7:",
              [(r["first_K"], r["cls"], f"{rel(r['rho_g'], r['rho_o']):.1e}") for r in rows], flush=True)
    l, r = configs.rig_calibs("hkust")
    for cid, c in DEPTH_CASES.items():
        tlc, trc, seed, _, _ = depth_inputs(cid)
        row = []
        for K in range(1, 11):
            vals = []
            for lib in (orc, prod):
                b = capi.Backend(lib, l, r, depth_params(c, lib, K))
                b.set_ts_pair(tlc, trc, np.eye(4))
                pts, ev = b.depth_solve(seed)
                b.close()
                vals.append([float(pts["inv_depth"][0]), float(pts["variance"][0]), float(pts["residual"][0]), int(ev)] if pts.size else None)
            row.append(vals)
        res["cases"][cid] = row
    json.dump(res, open(out, "w"), indent=1)


if __name__ == "__main__":
    main(sys.argv[1])
