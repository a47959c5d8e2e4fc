"""The depth LM's Student-t scale iteration on the device, case by case (util.DEPTH_CASES): esvo_depth_solve of the kernels
against the oracle's literal loop at max_iteration 1 (one Jacobian, at x0: the variance exposes ||J(x0)|| and the cost f at the
accepted point) and 10.  Cases whose evaluations tests/indep_depth.py finds rounding-decided are printed and counted, not
asserted.  With the parent's guard (r_min > 1e-6 alone) the band cases fail here at max_iteration 1, on rho or the variance:
67x1-band-1.5e-6, 67x1-rmin-0.99e-6 (its forward point has r_min 1.14e-6), 67x1-rmin-1.01e-6, 1x67-band-1.5e-6,
15x7-eps1e-08, 15x7-eps1e-06, 15x7-eps1e-6-rmin1.2e-6, 15x7-eps1e-6-rmin1e-5, 15x7-eps1e-8-rmin1e-4, 15x7-margin-accepted,
3x3-band, 113x1-band, 11x11-band and 127x1-band.  The regime is not read from the cost: a seed that solves its patch exactly
ends with a cost of 0 on one side and a few subnormal steps on the other."""
import numpy as np
import pytest

import indep_depth as idp
from esvo_b200 import capi, configs
from test_depth_irls_pins import HEPS, PL, PR, evaluations
from util import DEPTH_CASES, depth_inputs, depth_params, rel

pytestmark = pytest.mark.gpu
# Cases whose iterates part after the first step, measured with scripts/lm_tail_probe.py (DESIGN.md section 9):
#   flat    every residual is about -E and barely depends on rho, so the forward-difference Jacobian carries the residuals'
#           rounding-level differences into the step; rho parts by 3e-8 after one step and 2e-5 .. 5e-5 after ten, nfev agrees;
#   solved  the first step solves the patch: at that point the oracle's residuals are exactly 0 (cost 0) and the kernels' are
#           one ulp of a tap (a stall, cost ~1e-321), so the next Jacobian test (CosinusTooSmall) goes the other way; rho agrees
#           to 1e-15 but the evaluation counts differ from the second step on.
PARTING = {"15x7-nondeg-1pass": "flat", "15x7-nondeg-2pass": "flat", "15x7-c-above-0.95": "solved", "15x7-rmin-1e-7": "solved",
           "1x1-nondeg": "solved"}


def _solve(c, cid, lib, K):
    tl, tr, seed, _, _ = depth_inputs(cid)
    l, r = configs.rig_calibs("hkust")
    b = capi.Backend(lib, l, r, depth_params(c, lib, K))
    b.set_ts_pair(tl, tr, np.eye(4))
    pts, ev = b.depth_solve(seed)
    b.close()
    return pts, ev


@pytest.mark.parametrize("K", [1, 10])
@pytest.mark.parametrize("cid", list(DEPTH_CASES))
def test_depth_irls_case(oracle_lib, product_lib, cid, K):
    c = DEPTH_CASES[cid]
    po, evo = _solve(c, cid, oracle_lib, K)
    pg, evg = _solve(c, cid, product_lib, K)
    evs = [e for _, _, e in evaluations(cid)]
    if po.size:                                  # the accepted point and its forward point
        wx, wy = c["patch"]
        _, _, _, x, y = depth_inputs(cid)
        for rho in (float(po["inv_depth"][0]), float(po["inv_depth"][0]) * (1 + HEPS)):
            rv = idp.residual_vector(*depth_inputs(cid)[:2], PL, PR, x, y, rho, wx, wy)
            evs.append(None if rv is None else idp.evaluate(rv, wx * wy, c["nu"], c["scale"]))
    decided = not any(e is not None and e["rounding_decided"] for e in evs)
    line = (f"[depth irls {cid} K={K}] n {po.size}/{pg.size} nfev {evo}/{evg}; " +
            (f"rho {po['inv_depth'][0]:.17g}/{pg['inv_depth'][0]:.17g} var {po['variance'][0]:.6g}/{pg['variance'][0]:.6g} "
             f"cost {po['residual'][0]:.6g}/{pg['residual'][0]:.6g}" if po.size and pg.size else ""))
    print(line + ("" if decided else "  ROUNDING-DECIDED: regime only"))
    assert po.size == pg.size == 1
    co, cg = float(po["residual"][0]), float(pg["residual"][0])
    if not decided:
        # The pass at which a 5 % test passes is rounding-level (15x7-inside-margin-big: costs 1.8e-12 / 2.7e-13 measured on
        # an H100), but the regime is not: a reset there would give a cost near 1e3.
        assert co > 0 and cg > 0 and abs(np.log10(cg / co)) < 3, (co, cg)
        assert rel(pg["inv_depth"], po["inv_depth"]).max() <= 1e-7
        return
    # The oracle's literal cam2World can place the right patch one ulp (1.4e-14 px) away from the kernels' closed form, which
    # moves residuals of 1e-6 by 1e-8 relative.  Measured on an H100 at max_iteration 1, largest over the cases: rho 6e-8
    # (15x7-nondeg-2pass), variance 2e-7 (the shipped-nu cases), cost 8e-8 (costs below 1e-18 aside); at 10 the variance
    # grows to 2e-6.  The parent's guard moved the band cases' rho by 1e-7 .. 6e-6.
    part = PARTING.get(cid) if K > 1 else None
    if part == "flat":
        assert evo == evg and rel(pg["inv_depth"], po["inv_depth"]).max() <= 1e-4
        return
    if part != "solved":
        assert evo == evg
    assert rel(pg["inv_depth"], po["inv_depth"]).max() <= 1e-7, (po["inv_depth"][0], pg["inv_depth"][0])
    vo, vg = float(po["variance"][0]), float(pg["variance"][0])
    assert vo == vg or abs(vg - vo) <= (1e-6 if K == 1 else 1e-5) * abs(vo), (vo, vg)
    assert abs(cg - co) <= max(1e-6 * co, 1e-18), (co, cg)
