"""The event-to-event matcher's oracle (oracle/o_event_matcher.h) beyond the shipped configuration, on the case table of
tests/em_cases.py: against the independent numpy re-derivation (tests/indep_numpy.py::event_match), against closed-form
expectations where the table builds them (exact ties, the no-candidate-scored fallback, the epipolar bounds), against an
exact evaluation with mpmath, and through the capacity contract of the C ABI.  No GPU."""
import numpy as np
import pytest

import em_cases as E
from esvo_b200 import capi, configs

NUMPY_CASES = [cid for cid, c in E.CASES.items() if not c["boundary"]]
# |f64 cost - exact cost| over the accepted pairs of the natural and quarter-pixel cases, with the warp, the bilinear patches and
# the ZNCC evaluated at 50 digits from the same f64 inputs (measured <= 1.1e-14; see test_cost_is_within_bound_of_exact)
EXACT_COST_BOUND = 1e-13


@pytest.fixture(scope="module")
def oracle_for(oracle_lib):
    """oracle_for(rig): one oracle context per rig, holding the product's own tables for that rig."""
    cache = {}

    def get(rig):
        if rig not in cache:
            l, r = configs.rig_calibs(rig)
            be = capi.Backend(oracle_lib, l, r, E.params(rig, oracle_lib))
            lib = capi.load_product()
            for cam, c in ((0, l), (1, r)):
                be.set_rectify_tables(cam, *capi.compute_rectify_tables(lib, c))
            cache[rig] = be
        return cache[rig]
    return get


@pytest.fixture(scope="module")
def oracle_runs(oracle_for):
    """case id -> (inputs, kw, seeds, evals) of the oracle, computed once."""
    cache = {}

    def get(cid):
        if cid not in cache:
            c = E.CASES[cid]
            inp = E.case_inputs(c, oracle_for)
            kw = E.case_kw(c)
            be = E.load_case(oracle_for(inp["rig"]), inp)
            seeds, evals = E.run(be, inp, kw)
            cache[cid] = (inp, kw, seeds, evals, be.get_derived()["baseline"])
        return cache[cid]
    return get


@pytest.mark.parametrize("cid", NUMPY_CASES)
def test_oracle_vs_numpy(oracle_runs, cid):
    inp, kw, seeds, evals, baseline = oracle_runs(cid)
    ref, evals_ref = E.numpy_match(inp, kw, baseline)
    print(cid, "matches", seeds.size, "of", int(np.maximum(inp["counts"], 0).sum()), "evaluations", evals)
    assert seeds.size == len(ref) and evals == evals_ref
    for sd, m in zip(seeds, ref):
        assert sd["t_ns"] == m["t_ns"]
        assert np.array_equal(sd["x_left_raw"], [inp["left"]["x"][m["i"]], inp["left"]["y"][m["i"]]])
        assert np.array_equal(sd["x_left"], m["x_left"]) and np.array_equal(sd["x_right"], m["x_right"])
        assert abs(sd["cost"] - m["cost"]) < 1e-12
        if np.isinf(m["inv_depth"]):
            assert sd["inv_depth"] == m["inv_depth"]
        else:
            assert abs(sd["inv_depth"] - m["inv_depth"]) <= 4e-15 * abs(m["inv_depth"])
        assert np.array_equal(sd["T_world_virtual"].reshape(4, 4), m["T"])


def test_case_sizes(oracle_runs):
    """Every case that is meant to match something does; the wide patch and a zero time threshold (an empty window) match
    nothing and score nothing."""
    for cid in E.CASES:
        inp, kw, seeds, evals, _ = oracle_runs(cid)
        if cid in ("shape-wider-than-image", "fallback-ncc0.99", "win-zero-thr-small", "win-zero-thr-epoch"):
            assert seeds.size == 0 and evals == 0, cid
        else:
            assert seeds.size > 0, cid


@pytest.mark.parametrize("cid", ["ties-ncc0.5", "ties-ncc1"])
def test_exact_ties_pick_the_first_scoring_candidate(oracle_runs, cid):
    """Every scored candidate costs exactly 0.5; the winner is the first scoring candidate in time order, whichever lane and
    32-candidate pass of a warp-wide scan it falls in (k = 0, 5, 31, 32, 33, 70 failing candidates before it)."""
    inp, kw, seeds, evals, baseline = oracle_runs(cid)
    layout = E.tie_layout()
    assert seeds.size == len(layout)
    seeds = np.sort(seeds, order="t_ns")                                     # the output is thread-major
    assert evals == sum(n - k for k, n in layout)
    f = configs.rig_arrays("hkust")["left"]["P"][0, 0]
    for sd, (k, n) in zip(seeds, layout):
        d = 1 + k % 30                                                       # the candidate q = k
        assert sd["cost"] == 0.5
        assert sd["x_right"][0] == E.TIE_X - d + 0.25
        xl0 = E.TIE_X + 0.25
        assert sd["inv_depth"] == 1.0 / (baseline * f / (xl0 - (xl0 - d)))


def test_fallback_when_no_candidate_scores(oracle_runs):
    """min_cost stays 1: accepted with cost 1 at ncc_thr 1 (x_right of the first epipolar survivor, depth 0 -> rho = inf),
    rejected at 0.99."""
    inp, kw, seeds, evals, _ = oracle_runs("fallback-ncc1")
    assert seeds.size == 4 and evals == 0
    assert (seeds["cost"] == 1.0).all() and np.isposinf(seeds["inv_depth"]).all()
    assert (seeds["x_right"][:, 0] == 1.25).all() and (seeds["x_right"][:, 1] == 130.25).all()
    inp, kw, seeds, evals, _ = oracle_runs("fallback-ncc0.99")
    assert seeds.size == 0 and evals == 0


def test_epipolar_bounds(oracle_runs):
    """|dy| == epi_thr passes and nextafter(epi_thr, inf) fails; xr0 == xl0 fails and a disparity of one ulp passes (huge but
    finite depth); left LUT entries off the image are matched by the fallback only."""
    inp, kw, seeds, evals, _ = oracle_runs("epi-bounds")
    seeds = np.sort(seeds, order="t_ns")                                     # the output is thread-major
    xl = [tuple(s) for s in seeds["x_left"]]
    assert xl[:2] == [(100.25, 0.75), (100.25, 0.75)]                   # the two |dy| == 0.5 candidates; not the two ulp ones
    assert sorted(seeds["x_right"][:2, 1].tolist()) == [0.25, 1.25]
    assert (160.25, 0.75) in xl and (150.25, 0.75) not in xl
    s = seeds[[k for k, v in enumerate(xl) if v == (160.25, 0.75)][0]]
    assert 0 < s["inv_depth"] < 1e-12 and s["cost"] < 1.0
    off = seeds[seeds["x_left"][:, 0] < 0]
    assert off.size == 1 and off["cost"][0] == 1.0 and np.isposinf(off["inv_depth"][0])
    assert (seeds["x_left"][:, 0] > 346).sum() == 1
    assert seeds.size == 5


def test_capacity_contract(oracle_runs, oracle_for):
    """Too small a capacity returns ESVO_ERR_CAPACITY with the count; capacity 0 and no buffer is the count query."""
    inp, kw, seeds, evals, _ = oracle_runs("q-borders-15x7")
    be = oracle_for(inp["rig"])
    E.load_case(be, inp)
    assert E.em_match_raw(be, inp, kw, seeds.size - 1) == (-4, seeds.size, evals)
    assert E.em_match_raw(be, inp, kw, 0, with_buffer=False) == (-4, seeds.size, evals)
    assert E.em_match_raw(be, inp, kw, seeds.size) == (0, seeds.size, evals)


def test_case_table_reaches_every_branch(oracle_runs):
    """The decisions the table exists for, counted by the numpy re-derivation (tests/indep_numpy.py::event_match info)."""
    tot = {}
    reached = []
    for cid in NUMPY_CASES:
        inp, kw, _, _, baseline = oracle_runs(cid)
        info = {}
        E.numpy_match(inp, kw, baseline, info=info)
        for k, v in info.items():
            if isinstance(v, (int, np.integer)) and k not in ("total", "num_thread"):
                tot[k] = tot.get(k, 0) + int(v)
        reached.append((cid, info))
    print({k: v for k, v in tot.items()})
    winners = [w for _, i in reached for w in i["winners"]]
    assert any(lane != 0 and p >= 2 for lane, p in winners), "a winner beyond lane 0 in pass 2 or later"
    assert any(p >= 3 for _, p in winners)
    assert tot["ties"] > 0 and tot["fallback_accept"] > 0 and tot["fallback_reject"] > 0
    assert tot["epi_eq_accept"] > 0 and tot["epi_ulp_reject"] > 0 and tot["disp_zero_reject"] > 0 and tot["disp_ulp_accept"] > 0
    assert tot["on_low"] > 0 and tot["on_up"] > 0
    assert tot["patch_fail_far_y"] > 0 and tot["patch_fail_far_x"] > 0, "a warp that fails only through uly+wy >= H / ulx+wx >= W"
    assert tot["warp_fail"] > 0
    assert any(i["num_thread"] > i["total"] > 0 for _, i in reached), "NT > number of events"
    assert any(i["total"] > 256 and i["total"] % 256 for _, i in reached), "an em_order_kernel block boundary"
    assert any(i["num_thread"] == 1 for _, i in reached) and any(i["num_thread"] == 256 for _, i in reached)
    assert max(len(i["winners"]) + i["fallback_accept"] for _, i in reached) > 100


# ---- exact evaluation (mpmath, 50 digits) of warping2 -> patchInterpolation2 -> zncc_cost from the same f64 inputs ----------
def exact_warp(xl, inv, T_obs, T_rv, Pl, Pr):
    import mpmath as mp
    z = 1 / mp.mpf(inv)
    Pt = mp.matrix(4, 4)
    for i in range(3):
        for k in range(4):
            Pt[i, k] = mp.mpf(Pl[i, k])
    Pt[3, 3] = z
    ps = (mp.inverse(Pt) * z) * mp.matrix([mp.mpf(xl[0]), mp.mpf(xl[1]), 1, 1])
    p = [ps[i] / ps[3] for i in range(3)]
    T = mp.inverse(mp.matrix(T_obs.tolist())) * mp.matrix(T_rv.tolist())
    q = [sum(T[i, k] * p[k] for k in range(3)) + T[i, 3] for i in range(3)]
    out = []
    for P in (Pl, Pr):
        h = [sum(mp.mpf(P[i, k]) * q[k] for k in range(3)) + mp.mpf(P[i, 3]) for i in range(3)]
        out.append((h[0] / h[2], h[1] / h[2]))
    return out


def exact_cost(x1, x2, tl, tr, wx, wy):
    """None where the warp or a patch fails, otherwise the ZNCC cost, all at the working precision."""
    import mpmath as mp
    H, W = tl.shape
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    for x in (x1, x2):
        if x[0] < hx or x[0] > W - hx or x[1] < hy or x[1] > H - hy:
            return None
    patches = []
    for x, img in ((x1, tl), (x2, tr)):
        fx, fy = int(mp.floor(x[0])), int(mp.floor(x[1]))
        ulx, uly = fx - hx, fy - hy
        if ulx < 0 or uly < 0 or fx + hx >= W or fy + hy >= H or uly + wy >= H or ulx + wx >= W:
            return None
        q1, q2, q3, q4 = (fx + 1) - x[0], x[0] - fx, (fy + 1) - x[1], x[1] - fy
        s = img[uly:uly + wy + 1, ulx:ulx + wx + 1].astype(int).tolist()
        patches.append([q3 * (q1 * s[r][c] + q2 * s[r][c + 1]) + q4 * (q1 * s[r + 1][c] + q2 * s[r + 1][c + 1])
                        for r in range(wy) for c in range(wx)])
    a, b = patches
    n = len(a)
    ma, mb = mp.fsum(a) / n, mp.fsum(b) / n
    na = mp.sqrt(mp.fsum((v - ma) ** 2 for v in a)) + mp.mpf("1e-6")
    nb = mp.sqrt(mp.fsum((v - mb) ** 2 for v in b)) + mp.mpf("1e-6")
    return (1 - mp.fsum(((u - ma) / na) * ((v - mb) / nb) for u, v in zip(a, b))) / 2


EXACT_CASES = ("natural-epoch-hkust", "natural-epoch-dsec", "q-borders-15x7", "q-borders-16x6", "q-borders-2x2-moving", "win-epoch-shipped",
               "shape-16x6", "shape-31x3", "shape-25x5", "crowd-1200", "crowd-40", "rig-hkust", "rig-dsec", "rig-rpg", "rig-upenn", "nt7-total513", "nt2-total257",
               "slices-neg-above", "shape-2x2", "shape-1x15", "shape-15x1", "shape-176x3", "win-epoch")


def exact_cost_errors(runs, per_case=120):
    """|f64 cost - exact cost| of up to per_case accepted, scored seeds of every EXACT_CASES case."""
    import mpmath as mp
    mp.mp.dps = 50
    errs = []
    for cid in EXACT_CASES:
        inp, kw, seeds, _, _ = runs(cid)
        cams = configs.rig_arrays(inp["rig"])
        scored = seeds[seeds["cost"] < 1.0]
        for sd in scored[np.linspace(0, scored.size - 1, min(per_case, scored.size)).astype(int)] if scored.size else []:
            (x1, x2) = exact_warp(sd["x_left"], sd["inv_depth"], inp["T_obs"], sd["T_world_virtual"].reshape(4, 4), cams["left"]["P"],
                                  cams["right"]["P"])
            c = exact_cost(x1, x2, inp["tl"], inp["tr"], *kw["patch"])
            assert c is not None, cid
            errs.append(float(abs(mp.mpf(sd["cost"]) - c)))
    return np.array(errs)


def test_cost_is_within_bound_of_exact(oracle_runs):
    errs = exact_cost_errors(oracle_runs)
    print("pairs", errs.size, "max |f64 - exact|", errs.max(), "median", np.median(errs))
    assert errs.size >= 500
    assert errs.max() <= EXACT_COST_BOUND


def integer_rig_boundary_warps(runs):
    """(warps, warps whose exact x1 is integral, warps with an exact coordinate on a pixel boundary) over the epipolar
    survivors of the integer-rig cases (T_left_rv = I)."""
    import mpmath as mp
    mp.mp.dps = 50
    n = n_x1 = n_any = 0
    for cid, c in E.CASES.items():
        if not c["boundary"]:
            continue
        inp, kw, _, _, baseline = runs(cid)
        cams = configs.rig_arrays(inp["rig"])
        f = cams["left"]["P"][0, 0]
        L, R = inp["left"], inp["right"]
        lo, hi = 0, 0
        for i in range(L["x"].size):
            xl = inp["lut_l"][L["y"][i], L["x"][i]]
            for j in np.nonzero(np.abs(R["t"] - L["t"][i]) < 5_000_000)[0]:
                xr = inp["lut_r"][R["y"][j], R["x"][j]]
                if not (abs(xl[1] - xr[1]) <= kw["epi_thr"] and xr[0] < xl[0]):
                    continue
                inv = 1.0 / (baseline * f / (xl[0] - xr[0]))
                (x1, x2) = exact_warp(xl, inv, inp["T_obs"], inp["poses"][0].reshape(4, 4), cams["left"]["P"], cams["right"]["P"])
                n += 1
                on = [abs(v - mp.nint(v)) < mp.mpf("1e-40") for v in (*x1, *x2)]     # integral up to the 50-digit rounding
                n_x1 += int(on[0] and on[1])
                n_any += int(any(on))
    return n, n_x1, n_any


def test_integer_rig_warps_sit_on_pixel_boundaries(oracle_runs):
    n, n_x1, n_any = integer_rig_boundary_warps(oracle_runs)
    print("integer-rig warps", n, "exact x1 integral", n_x1, "any coordinate integral", n_any)
    assert n > 1000 and n_x1 == n
