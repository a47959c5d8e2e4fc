"""The Student-t scale iteration of the depth LM on hand-built residual vectors (util.DEPTH_CASES), without a GPU: the oracle
against the scalar restatement tests/indep_depth.py to the bit, the table's reach over the iteration's arms, and an exhaustive
check of the degenerate-regime guard (DESIGN.md deviation 4) against the reference's literal loop."""
import ctypes as C
import math

import numpy as np
import pytest

import indep_depth as idp
from esvo_b200 import capi, configs
from util import DEPTH_CASES, depth_inputs, depth_params

HEPS = 1.4901161193847656e-08
_A = configs.rig_arrays("hkust")
PL, PR = _A["left"]["P"], _A["right"]["P"]


def case_evaluations(cid):
    """The restatement at the seed's x0 and at x0 + h (NumericalDiff's forward point): [(rho, r or None, evaluate(r) or None)]."""
    c = DEPTH_CASES[cid]
    tl, tr, seed, x, y = depth_inputs(cid)
    wx, wy = c["patch"]
    out = []
    x0 = float(seed["inv_depth"][0])
    for rho in (x0, x0 + HEPS * abs(x0)):
        r = idp.residual_vector(tl, tr, PL, PR, x, y, rho, wx, wy)
        out.append((rho, r, None if r is None else idp.evaluate(r, wx * wy, c["nu"], c["scale"])))
    return out


_EVALS = {}


def evaluations(cid):
    if cid not in _EVALS:
        _EVALS[cid] = case_evaluations(cid)
    return _EVALS[cid]


@pytest.mark.parametrize("cid", list(DEPTH_CASES))
def test_oracle_matches_sequential_restatement(oracle_lib, cid):
    """DepthProblem::operator() of the oracle, which runs the reference's literal loop, against the restatement's sequential
    run at x0 and x0 + h: the same regime (a stall at a subnormal scale leaves every |f| below 1e-150), the failed-warp value
    to the bit, and f within 1e-7 relative elsewhere (the oracle's cam2World may place the right patch one ulp away from the
    restatement's, which moves residuals of 1e-6 by 1e-8 relative)."""
    c = DEPTH_CASES[cid]
    tl, tr, seed, _, _ = depth_inputs(cid)
    l, r = configs.rig_calibs("hkust")
    o = capi.Backend(oracle_lib, l, r, depth_params(c, oracle_lib))
    o.set_ts_pair(tl, tr, np.eye(4))
    fn = oracle_lib.lib.esvo_oracle_op_depth_residual
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.POINTER(C.c_double)]
    fn.restype = C.c_int
    N = c["patch"][0] * c["patch"][1]
    for rho, rv, ev in evaluations(cid):
        fo = np.zeros(N)
        ok = fn(o.ctx, seed.ctypes.data_as(C.c_void_p), rho, fo.ctypes.data_as(C.POINTER(C.c_double)))
        assert ok == (rv is not None), (cid, rho)
        if rv is None:
            assert fo.tobytes() == np.full(N, idp.failed_value(c["nu"], c["scale"])).tobytes(), cid
            continue
        want = np.array(ev["f"])
        assert (np.abs(fo).max() < 1e-150) == (ev["seq"]["kind"] == "stall"), (cid, rho, ev["seq"]["kind"])
        if ev["seq"]["kind"] != "stall":
            assert np.all(np.abs(fo - want) <= 1e-7 * np.abs(want)), (cid, rho, np.abs(fo - want).max())


def test_case_table_reaches_every_arm():
    """Over the table's evaluations the loop ends through sum == 0, through the 5 % test at a normal scale after 1, 2 and
    >= 10 passes, and through the 5 % test at a subnormal scale (a stall); it passes 1e-30 and 1e-250; both weight paths are
    taken; the parent's guard accepts vectors whose literal loop stalls, the fixed guard accepts others and declines those;
    the warp fails at x0 + h only; and a case sits one ulp either side of the guard's 1e-9 margin.

    Two arms no input reaches, so the table does not claim them:
      * sum == 0 above 1e-30 (and above 1e-250): every term is r^2 (nu+1) s / (nu s + r^2) with s > 1e-250, which is 0 only if
        r^2 is 0 or underflows; then every non-zero residual is below 1.5e-154 and the vector is degenerate with
        min r^2 = 0 for lm_kernel, so the loop runs -- but the terms stay 0 at every scale, and the first pass resets: at the
        starting scale td_scale^2, i.e. in the fast arm only when all a^2 are 0.  That vector has nz = 0 and c = 0, which the
        guard takes (gap * min r^2 = 0.95 N * 1e300).
      * the 5 % test passed between 1e-250 and 1e-30: a fixed point s* of the update below 1e-30 needs every non-zero
        r^2 (nu+1) / (nu + r^2 / s*) ~ (nu+1) s*, i.e. every residual below about sqrt(s*) < 1e-15 -- far below ulp(255), the
        rounding of a bilinear tap of an 8-bit surface, so no patch produces it; a degenerate vector never converges."""
    seen = dict(kinds=set(), passes=set(), below30=False, below250=False, subnormal=False, paths=set(), failed=0,
                old_only=0, new=0, rounding=[])
    for cid in DEPTH_CASES:
        for rho, rv, ev in evaluations(cid):
            if rv is None:
                seen["failed"] += 1
                continue
            s = ev["seq"]
            seen["kinds"].add(s["kind"])
            if s["kind"] == "converged":
                seen["passes"].add(min(s["passes"], 10))
            for k in ("below30", "below250", "subnormal"):
                seen[k] |= s[k] or ev["dev"][k]
            seen["paths"].add(ev["path"])
            seen["old_only"] += ev["shortcut_old"] and not ev["shortcut_new"] and s["kind"] == "stall"
            seen["new"] += ev["shortcut_new"]
            if ev["rounding_decided"]:
                seen["rounding"].append(cid)
            assert not ev["shortcut_new"] or s["kind"] == "reset", cid
    print({k: v for k, v in seen.items()})
    assert seen["kinds"] == {"reset", "converged", "stall"}
    assert {1, 2, 10} <= seen["passes"]
    assert seen["below30"] and seen["below250"] and seen["subnormal"]
    assert seen["paths"] == {"reciprocal", "division"}
    assert seen["failed"] == 1 and seen["old_only"] >= 10 and seen["new"] >= 10
    assert [c for c in DEPTH_CASES if DEPTH_CASES[c].get("ulp_at")] == ["15x7-margin-accepted", "15x7-margin-declined"]
    ev_a = evaluations("15x7-margin-accepted")[0][2]
    ev_d = evaluations("15x7-margin-declined")[0][2]
    assert ev_a["shortcut_old"] and not ev_d["shortcut_old"]


def test_planted_mistakes_are_caught():
    """Which case catches each planted mistake in the kernels' scale iteration (tests/test_gpu_depth_irls.py runs the cases on
    the device; here the restatement shows that the mistake changes the outcome of the case's evaluation at x0).

      * the (1 - 1e-9) margin dropped from irls_degenerate: 15x7-inside-margin-big.  c is one ulp below 0.95 and 33 residuals
        of about -10 pass gap * min r^2 >= 2^-49 N, so without the margin the kernels take the reset (|f| ~ 10); with it both
        loops end through a 5 % test near a scale of 1e-14 (|f| ~ 2e-7).  The pass at which that test passes is decided at
        rounding level, so the device parity checks this case for its regime, not its value.
      * ">=" for ">" in the division arm's 5 % test: 67x1-stall-at-exact-5pct.  Its last subnormal step shrinks the scale by
        exactly 1/20 (a whole number of 2^-1074 steps, so (s1 - s2) / s1 rounds to the same double as 0.05); ">" stops there,
        ">=" takes one more step and stalls at another scale (|f| moves by about 10 %).
      * "<" for "<=" in lm2_kernel's tiny test (|r| <= 1e-6): outcome-equivalent.  The ballot of tiny residuals is read only
        where gap >= 2^-49 / 1e-12 N; there a vector whose smallest residual is exactly 1e-6 has gap * min r^2 >= 2^-49 N, so
        the literal loop it runs instead of the shortcut provably resets: the same scale, the same f, only slower.
      * 1e-300 for 1e-200 in the weight switch: outcome-equivalent, because no evaluation ends with a scale in (1e-300, 1e-200].
        Resets end at td_scale^2; a 5 % exit at a normal scale below 1e-30 needs a fixed point there, i.e. every residual below
        about 1e-15 (see test_case_table_reaches_every_arm); every other exit is a stall at a subnormal scale.  Both weight forms
        are within rounding of each other at any normal scale above 1e-300 anyway.
    """
    N = 105
    c = DEPTH_CASES["15x7-inside-margin-big"]
    _, rv, ev = evaluations("15x7-inside-margin-big")[0]
    nzr = [v for v in rv if v != 0]
    gap = 0.95 * N - (c["nu"] + 1) * len(nzr)
    assert (c["nu"] + 1) * len(nzr) < 0.95 * N and not idp.degenerate(len(nzr), N, c["nu"])
    assert gap * min(v * v for v in nzr) >= idp.RESET_GAP * N          # the guard without its margin would take the reset
    assert ev["seq"]["kind"] == ev["dev"]["kind"] == "converged" and ev["seq"]["sc2"] < 1e-12
    c = DEPTH_CASES["67x1-stall-at-exact-5pct"]
    _, rv, ev = evaluations("67x1-stall-at-exact-5pct")[0]
    mutant = idp.scale_loop_dev(rv, 67, c["nu"], c["scale"], div_ge=True)
    assert ev["dev"]["kind"] == "stall" and not ev["rounding_decided"]
    assert mutant["sc2"] != ev["dev"]["sc2"]


def test_guard_sweep_proves_reset():
    """Wherever the fixed guard takes the shortcut, the reference's literal loop resets the scale (sum == 0).  The grid: patch
    sizes 1, 9, 20, 67, 105, 113, 127 and 128; for each, nz = 1, 2, 3, half and the largest two degenerate counts (not every
    nz: the loop runs about 14 000 passes near the threshold, and the bound depends on nz only through gap); eps from just
    above the 1e-9 margin to 0.1; min |r| at the guard's edge and at 1.5 x it; vectors of equal residuals and vectors mixing
    the smallest residual with larger ones up to 100."""
    rng = np.random.default_rng(5)
    rows, meta = [], []
    for N in (1, 9, 20, 67, 105, 113, 127, 128):
        for eps in (1.5e-9, 1e-8, 1e-7, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 0.1):
            nz_max = int(0.95 * N / 1.0)
            for nz in sorted({1, 2, 3, max(1, nz_max // 2), max(1, nz_max - 1), max(1, nz_max)}):
                nu = 0.95 * N * (1 - eps) / nz - 1
                if nu <= 0 or not idp.degenerate(nz, N, nu):
                    continue
                gap = 0.95 * N - (nu + 1) * nz
                for k in (1.0, 1.5):
                    rmin = math.sqrt(k * idp.RESET_GAP * N / gap)
                    for mixed in (False, True):
                        r = np.zeros(N)
                        pos = rng.choice(N, nz, replace=False)
                        r[pos] = rmin
                        if mixed and nz > 1:
                            r[pos[1:]] = rmin * np.exp(rng.uniform(0, math.log(100 / rmin), nz - 1))
                        while not idp.shortcut_new(list(r), N, nu):  # rounding of rmin at the edge: move it up by ulps
                            r[r == r[pos[0]]] = np.nextafter(r[pos[0]], 1)
                        assert idp.shortcut_new(list(r), N, nu)
                        rows.append((N, nu, r))
                        meta.append((N, nz, eps, k, mixed, idp.shortcut_old(list(r), N, nu)))
    bad, old_bad = [], 0
    for N in sorted({m[0] for m in meta}):
        for nu in sorted({row[1] for row in rows if row[0] == N}):
            idx = [i for i, row in enumerate(rows) if row[0] == N and row[1] == nu]
            kind, _ = idp.reset_batch(np.stack([rows[i][2] for i in idx]), nu, 17.277)
            for i, kd in zip(idx, kind):
                if kd != 0:
                    bad.append(meta[i])
    print(f"{len(rows)} vectors at the fixed guard's edge; parent guard accepted {sum(m[5] for m in meta)} of them")
    assert not bad, bad[:10]


def test_parent_guard_accepts_stalling_vectors():
    """The defect the fixed guard removes: at 67 x 1 with 20 residuals of 1.5e-6 and the shipped dsec nu (eps = 1.6e-4) the
    parent's guard took the shortcut (reset, |f| ~ 1.8e-6) where the literal loop stalls at a subnormal scale after 13 718 passes
    (|f| ~ 2e-160); the fixed guard declines it."""
    r = [1.5e-6] * 20 + [0.0] * 47
    ev = idp.evaluate(r, 67, 2.182, 17.277)
    assert ev["shortcut_old"] and not ev["shortcut_new"]
    assert ev["seq"]["kind"] == ev["dev"]["kind"] == "stall" and ev["seq"]["passes"] == 13718
    assert max(abs(v) for v in ev["f"]) < 1e-159 and not ev["rounding_decided"]
