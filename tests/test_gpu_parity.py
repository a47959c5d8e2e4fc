"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle on identical
inputs.  Integer/index outputs must be bit-exact; f64 outputs within 1e-4 relative (north_star),
in practice ~1e-9."""
import numpy as np
import pytest

from esvo_b200 import capi, configs, synth
from util import (TRACK_CASES, bits_equal, build_ts_pair, fold_replay, fold_vector, grid_vs_map, make_backends, maps_bit_identical, rel, scenario, track_backend,
                  track_inputs, track_params, track_trace)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rig", ["hkust", "dsec"])
def test_time_surface_bit_exact(oracle_lib, product_lib, rig):
    s = scenario(rig)
    o, g = make_backends(rig, oracle_lib, product_lib)
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        n = e["x"].size
        # push in three uneven batches
        cuts = [0, n // 3, n // 3 + 7, n]
        for a, b in zip(cuts[:-1], cuts[1:]):
            for be in (o, g):
                be.ts_push_events(cam, e["x"][a:b], e["y"][a:b], e["t"][a:b], e["p"][a:b])
        for T in (s["t_ts_ns"], int(e["t"][n // 2]), int(e["t"][n - 50]), int(e["t"][0])):
            io, to = o.ts_build(cam, T)
            ig, tg = g.ts_build(cam, T)
            assert np.array_equal(io, ig), f"idx grid differs cam{cam} T={T}: {(io != ig).sum()} px"
            assert np.array_equal(to, tg), f"TS image differs cam{cam} T={T}: {(to != tg).sum()} px"
        assert (to >= 0).all()


@pytest.mark.parametrize("order", ["txyp", "xytp", "pad"])
def test_time_surface_packet_buffer_push(oracle_lib, product_lib, order):
    """Host pushes whose four arrays are adjacent in memory (one packet buffer) take the single-copy path of ts_push; arrays in
    separate allocations take four copies.  Same bytes either way, for any order of the arrays inside the packet and with a
    misaligned packet start."""
    s = scenario("hkust")
    o, g = make_backends("hkust", oracle_lib, product_lib)
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        n = e["x"].size
        half = n // 2
        for a, b in ((0, half), (half, n)):
            m = b - a
            lead = 8 if order == "pad" else 0
            buf = np.zeros(13 * m + 64, np.uint8)
            if order == "xytp":
                ox, oy = lead, lead + 2 * m
                ot = (oy + 2 * m + 7) // 8 * 8
                op = ot + 8 * m
            else:
                ot = lead
                ox = ot + 8 * m; oy = ox + 2 * m; op = oy + 2 * m
            x = buf[ox:ox + 2 * m].view(np.uint16); y = buf[oy:oy + 2 * m].view(np.uint16)
            t = buf[ot:ot + 8 * m].view(np.int64); p = buf[op:op + m]
            x[:] = e["x"][a:b]; y[:] = e["y"][a:b]; t[:] = e["t"][a:b]; p[:] = e["p"][a:b]
            g.ts_push_events(cam, x, y, t, p)                    # one packet
            o.ts_push_events(cam, e["x"][a:b], e["y"][a:b], e["t"][a:b], e["p"][a:b])
        for T in (s["t_ts_ns"], int(e["t"][n - 50])):
            io, to = o.ts_build(cam, T)
            ig, tg = g.ts_build(cam, T)
            assert np.array_equal(io, ig) and np.array_equal(to, tg), (order, cam, T)


def test_time_surface_queue_depth_quirk(oracle_lib, product_lib):
    """A pixel with >= max_event_queue_len events newer than T yields 'no event' (TimeSurface.h:52-75)."""
    o, g = make_backends("hkust", oracle_lib, product_lib)
    n = 60
    x = np.full(n, 100, np.uint16); y = np.full(n, 80, np.uint16)
    t = (1_000_000_000 + np.arange(n) * 1000).astype(np.int64); p = np.ones(n, np.uint8)
    x[::7] = 101
    for be in (o, g):
        be.ts_push_events(0, x, y, t, p)
    for T in (int(t[5]), int(t[30]), int(t[45]), int(t[-1]) + 1):
        io, to = o.ts_build(0, T)
        ig, tg = g.ts_build(0, T)
        assert np.array_equal(io, ig) and np.array_equal(to, tg)


def test_polarity_mode_bit_exact(oracle_lib, product_lib):
    s = scenario("hkust")
    def tw(p):
        p.ignore_polarity = 0
    o, g = make_backends("hkust", oracle_lib, product_lib, tweak=tw)
    e = s["left"]
    for be in (o, g):
        be.ts_push_events(0, e["x"], e["y"], e["t"], e["p"])
    io, to = o.ts_build(0, s["t_ts_ns"]); ig, tg = g.ts_build(0, s["t_ts_ns"])
    assert np.array_equal(io, ig) and np.array_equal(to, tg)


@pytest.mark.parametrize("rig,median,polarity", [("hkust", 1, 1), ("hkust", 0, 0), ("upenn", 1, 1), ("dsec", 1, 1)])
def test_time_surface_forward_mode_bit_exact(oracle_lib, product_lib, rig, median, polarity):
    """FORWARD mode (TimeSurface.cpp:86-116): bilinear splat onto the rectified grid with a clamp after every
    accumulation -- order-dependent, replayed in the reference's raster order on the device."""
    s = scenario(rig)
    def tw(p):
        p.time_surface_mode = 1; p.median_blur_kernel_size = median; p.ignore_polarity = polarity
    o, g = make_backends(rig, oracle_lib, product_lib, tweak=tw)
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        for be in (o, g):
            be.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
        n = e["x"].size
        for T in (s["t_ts_ns"], int(e["t"][n // 2])):        # fast path and general (older T) path
            io, to = o.ts_build(cam, T)
            ig, tg = g.ts_build(cam, T)
            assert np.array_equal(io, ig)
            assert np.array_equal(to, tg), f"forward TS differs cam{cam} T={T}: {(to != tg).sum()} px"
        assert len(np.unique(to)) > 10                       # a real image, with saturated accumulations in it
    # the clamp at 1 must have been exercised (several events landing on the same rectified pixel)
    assert (to == 255).any()


def test_time_surface_unordered_stamps(oracle_lib, product_lib):
    """Out-of-order stamps with esvo_ts_set_unordered_input: the device prefix scan (running arg-max of the stamps,
    carried across pushes) reproduces the reference's events_.back() behaviour bit for bit; without the switch the
    violation is reported."""
    s = scenario("hkust")
    o, g = make_backends("hkust", oracle_lib, product_lib)
    e = s["left"]
    rng = np.random.default_rng(9)
    t = e["t"].copy()
    late = rng.random(t.size) < 0.08                       # 8 % of the events arrive with a stamp up to 2 ms in the past
    t[late] -= rng.integers(1_000, 2_000_000, late.sum())
    t[0] = e["t"][0]
    assert (np.diff(t) < 0).sum() > 100
    g.ts_set_unordered_input(0, True)
    n = t.size
    cuts = [0, 700, 701, 1024, 5000, n // 2, n]              # batch boundaries inside / across scan blocks
    for a, b in zip(cuts[:-1], cuts[1:]):
        for be in (o, g):
            be.ts_push_events(0, e["x"][a:b], e["y"][a:b], t[a:b], e["p"][a:b])
    for T in (int(t.max()) + 1, int(np.sort(t)[n // 2]), int(np.sort(t)[n - 100])):
        io, to = o.ts_build(0, T)
        ig, tg = g.ts_build(0, T)
        assert np.array_equal(io, ig), f"idx grid differs T={T}: {(io != ig).sum()} px"
        assert np.array_equal(to, tg)
    # default mode: the same input is rejected, not silently mis-handled
    g.ts_set_unordered_input(1, False)
    g.ts_push_events(1, e["x"][:5000], e["y"][:5000], t[:5000], e["p"][:5000])
    with pytest.raises(capi.EsvoError):
        g.ts_build(1, int(t.max()) + 1)


def _bm_pair(oracle_lib, product_lib, rig, tweak=None):
    s = scenario(rig)
    o, g = make_backends(rig, oracle_lib, product_lib, tweak=tweak)
    tl, tr = build_ts_pair(o, s)
    for be in (o, g):
        be.set_ts_pair(tl, tr, s["T_world_left"])
    sd = s["seeds"]
    so, evo = o.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    sg, evg = g.bm_match(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    return s, o, g, so, sg, evo, evg


def _tweak(**kw):
    def tw(p):
        for k, v in kw.items():
            setattr(p, k, v)
    return tw


def bm_branches(p, dmin, dmax):
    """The kernel(s) of bm_run (esvo_b200/csrc/bm.cu, bm_run) a parameter set reaches, as tags.  The rule is a copy of
    bm_run's dispatch: the TMA kernel takes step 1, left-right rigs with wy <= 8 and a strip wx + dmax - dmin + 15 <= 112
    (box 64 up to 64 bytes, else 112); everything else runs bm_kernel, for each of the reasons listed."""
    wx, wy, step = p.patch_size_x, p.patch_size_y, max(1, p.bm_step)
    if dmax < dmin:
        return {"empty"}
    strip = wx + dmax - dmin + 15
    if step == 1 and not p.bm_updown and wy <= 8 and strip <= 112:
        return {"tma64" if strip <= 64 else "tma112"}
    tags = set()
    if step > 1:
        tags.add("ldg:step")
        if dmin == 0:
            tags.add("ldg:step-dmin0")      # the reference's size_t fine-search start wraps below 0 (EventBM.cpp:128)
    if p.bm_updown:
        tags.add("ldg:updown")
    if wy > 8:
        tags.add("ldg:wy>8")
    if strip > 112:
        tags.add("ldg:strip>112")
    if (dmax - dmin) // step + 1 > 192:
        tags.add("ldg:>192-candidates")     # the j < BM_MAXC guard of the coarse cost map
    return tags


BM_BRANCHES = {"tma64", "tma112", "ldg:step", "ldg:step-dmin0", "ldg:updown", "ldg:wy>8", "ldg:strip>112", "ldg:>192-candidates", "empty"}

# (id, rig, parameter changes, intended (dmin, dmax), floor on the accepted seeds).  hkust: f b = 13.86 px, so the derived range is
# [max(floor(13.86 rmin), bm_min), min(ceil(13.86 rmax), bm_max)] = [3, 28] by default; dsec: f b = 319.9 px, [0, 80].
BM_CASES = [
    ("hkust", "hkust", {}, (3, 28), 400),
    ("dsec", "dsec", {}, (0, 80), 100),
    ("hkust-strip64", "hkust", dict(invdepth_max_range=3.0, bm_max_disparity=37), (3, 37), 400),
    ("hkust-strip65", "hkust", dict(invdepth_max_range=3.0, bm_max_disparity=38), (3, 38), 400),
    ("hkust-strip112", "hkust", dict(invdepth_max_range=7.0, bm_max_disparity=85), (3, 85), 400),
    ("hkust-strip113", "hkust", dict(invdepth_max_range=7.0, bm_max_disparity=86), (3, 86), 400),
    ("hkust-32cand", "hkust", dict(invdepth_max_range=3.0, bm_max_disparity=34), (3, 34), 400),
    ("hkust-33cand", "hkust", dict(invdepth_max_range=3.0, bm_max_disparity=35), (3, 35), 400),
    ("hkust-198cand", "hkust", dict(invdepth_max_range=15.0, bm_max_disparity=200), (3, 200), 400),
    ("hkust-3x3", "hkust", dict(patch_size_x=3, patch_size_y=3), (3, 28), 500),
    ("hkust-5x5", "hkust", dict(patch_size_x=5, patch_size_y=5), (3, 28), 500),
    ("hkust-25x5", "hkust", dict(patch_size_x=25, patch_size_y=5), (3, 28), 300),
    ("hkust-7x15", "hkust", dict(patch_size_x=7, patch_size_y=15), (3, 28), 400),
    ("hkust-9x9", "hkust", dict(patch_size_x=9, patch_size_y=9), (3, 28), 400),
    ("hkust-127x1", "hkust", dict(patch_size_x=127, patch_size_y=1), (3, 28), 80),
    ("hkust-1x127", "hkust", dict(patch_size_x=1, patch_size_y=127), (3, 28), 40),
    ("hkust-41x3", "hkust", dict(patch_size_x=41, patch_size_y=3), (3, 28), 250),
    ("hkust-step2", "hkust", dict(bm_step=2), (3, 28), 300),
    ("hkust-step3", "hkust", dict(bm_step=3), (3, 28), 200),
    ("hkust-step5", "hkust", dict(bm_step=5), (3, 28), 150),
    ("dsec-step2", "dsec", dict(bm_step=2), (0, 80), 400),
    ("dsec-step3", "dsec", dict(bm_step=3), (0, 80), 400),
    ("dsec-step5", "dsec", dict(bm_step=5), (0, 80), 400),
    ("hkust-updown", "hkust", dict(bm_updown=1), (3, 28), 40),
    ("hkust-empty", "hkust", dict(bm_min_disparity=30, bm_max_disparity=20), (30, 20), 0),
]


def _bm_case_params(rig, kw, lib):
    p = configs.params_for(rig, lib)
    _tweak(**kw)(p)
    return p


def test_block_matching_cases_cover_every_bm_run_branch(oracle_lib):
    seen = set()
    for name, rig, kw, (dmin, dmax), floor in BM_CASES:
        seen |= bm_branches(_bm_case_params(rig, kw, oracle_lib), dmin, dmax)
    assert seen == BM_BRANCHES, BM_BRANCHES - seen


@pytest.mark.parametrize("rig,kw,rng,floor", [pytest.param(*c[1:], id=c[0]) for c in BM_CASES])
def test_block_matching_parity(oracle_lib, product_lib, rig, kw, rng, floor):
    s, o, g, so, sg, evo, evg = _bm_pair(oracle_lib, product_lib, rig, tweak=_tweak(**kw))
    for be in (o, g):
        d = be.get_derived()
        assert (d["min_disparity"], d["max_disparity"]) == rng, d
    kern = sorted(bm_branches(o.params, *rng))
    print(f"[bm {rig} {kw}] kernel {kern}: seeds oracle {so.size} gpu {sg.size}, evaluations {evo} / {evg}, "
          f"max |cost diff| {np.abs(so['cost'] - sg['cost']).max() if so.size == sg.size and so.size else 0:.1e}")
    if floor == 0:
        assert so.size == sg.size == 0 and evo == evg == 0
        return
    assert so.size > floor
    assert evo == evg, "number of zncc evaluations differs"
    assert so.size == sg.size, f"accept sets differ: {so.size} vs {sg.size}"
    assert np.array_equal(so["x_left_raw"], sg["x_left_raw"])      # same events, same (thread-major) order
    assert np.array_equal(so["x_left"], sg["x_left"])
    assert np.array_equal(so["t_ns"], sg["t_ns"])
    assert np.array_equal(so["T_world_virtual"], sg["T_world_virtual"])
    # integer work: the disparity must be EQUAL (a mismatch could only come from an exact tie of the f64 cost, DESIGN.md deviation 1)
    assert np.array_equal(so["disp"], sg["disp"]), f"{(so['disp'] != sg['disp']).sum()} disparity mismatches"
    assert np.abs(so["cost"] - sg["cost"]).max() < 1e-12
    assert np.array_equal(so["inv_depth"], sg["inv_depth"]) and np.array_equal(so["x_right"], sg["x_right"])


def test_block_matching_coarse_to_fine(oracle_lib, product_lib):
    def tw(p):
        p.bm_step = 3
    s, o, g, so, sg, evo, evg = _bm_pair(oracle_lib, product_lib, "hkust", tweak=tw)
    assert so.size > 50 and evo == evg and so.size == sg.size
    assert np.array_equal(so["x_left_raw"], sg["x_left_raw"])
    assert np.array_equal(so["disp"], sg["disp"])


def lm_kernel_for(lsnorm, wx, wy):
    """The instantiation lm_run (esvo_b200/csrc/lm.cu) launches: Tdist with m = wx wy <= 112 runs lm2_kernel<7, 20>, larger
    patches the 8-slot lm_kernel; l2 and zncc run lm_kernel with 7 or 8 slots per lane by the same bound."""
    slots = 7 if wx * wy <= 7 * 16 else 8
    if lsnorm == capi.LSNORM_TDIST:
        return "lm2_kernel<7,20>" if slots == 7 else "lm_kernel<8,true>"
    return f"lm_kernel<{slots},false>"


_TD, _L2, _ZN = capi.LSNORM_TDIST, capi.LSNORM_L2, capi.LSNORM_ZNCC
# (rig, norm, patch, floor on the solved seeds).  The first four ids are the 15 x 7 cases of the shipped yamls.
LM_CASES = [pytest.param("hkust", _TD, (15, 7), 600, id="hkust-1"), pytest.param("dsec", _TD, (15, 7), 900, id="dsec-1"),
            pytest.param("hkust", _L2, (15, 7), 600, id="hkust-0"), pytest.param("hkust", _ZN, (15, 7), 600, id="hkust-2")]
LM_CASES += [pytest.param("hkust", _TD, (wx, wy), 600, id=f"hkust-1-{wx}x{wy}")
             for wx, wy in ((1, 1), (3, 3), (15, 1), (1, 15), (5, 5), (17, 5), (7, 15), (37, 3),             # lm2_kernel
                            (113, 1), (23, 5), (13, 9), (17, 7), (11, 11), (127, 1))]                      # lm_kernel<8, ...>
LM_CASES += [pytest.param("hkust", norm, (wx, wy), 600, id=f"hkust-{norm}-{wx}x{wy}") for norm in (_L2, _ZN) for wx, wy in ((5, 5), (11, 11))]


@pytest.mark.parametrize("rig,lsnorm,patch,floor", LM_CASES)
def test_depth_solver_parity(oracle_lib, product_lib, rig, lsnorm, patch, floor):
    """Seeds of the default 15 x 7 block matching into solvers created with the patch shape and norm under test (the seed
    does not depend on the shape): every LM instantiation lm_run picks by shape and norm, incl. patches of one row or one
    column, m < 16 (lanes without a residual slot) and m at the 112 / 128 bounds."""
    s, o, g, so, sg, _, _ = _bm_pair(oracle_lib, product_lib, rig)
    if patch != (15, 7) or lsnorm != _TD:
        o, g = make_backends(rig, oracle_lib, product_lib, tweak=_tweak(lsnorm=lsnorm, patch_size_x=patch[0], patch_size_y=patch[1]))
        tl, tr = build_ts_pair(o, s)
        for be in (o, g):
            be.set_ts_pair(tl, tr, s["T_world_left"])
    po, evo = o.depth_solve(so)
    pg, evg = g.depth_solve(so)           # identical seeds into both solvers
    assert po.size > floor
    assert po.size == pg.size, f"solved sets differ: {po.size} vs {pg.size}"
    assert np.array_equal(po["x"], pg["x"]) and np.array_equal(po["row"], pg["row"]) and np.array_equal(po["col"], pg["col"])
    r = rel(pg["inv_depth"], po["inv_depth"])
    print(f"[lm {rig} norm {lsnorm} {patch[0]}x{patch[1]}] {lm_kernel_for(lsnorm, *patch)}: n={po.size} of {so.size} seeds, "
          f"rho rel err max {r.max():.3e} median {np.median(r):.3e}; nfev oracle {evo} gpu {evg}")
    w = int(np.argmax(r))
    print(f"   worst seed #{w}: x_left {po['x'][w]}, rho oracle {po['inv_depth'][w]:.9g} gpu {pg['inv_depth'][w]:.9g}, cost {po['residual'][w]:.6g} / {pg['residual'][w]:.6g}")
    # The shipped 15 x 7 shape keeps the full bar.  Off it, 1 - 3 of ~760 seeds (flat problems, or patches that leave the image
    # during the iterations) end their forward-difference LM on a different iterate, and on a few converged seeds the
    # variance / cost differ beyond the bar; the median stays at 1e-9 (DESIGN.md section 9, open lead).  The failed-warp value
    # these cases cannot pin is checked exactly by test_depth_solver_failed_warp_value.
    shipped = patch == (15, 7)
    assert (r < 1e-4).mean() >= (0.999 if shipped else 0.995), f"{(r >= 1e-4).sum()} of {r.size} seeds beyond 1e-4"
    assert np.median(r) < 1e-7   # forward-difference Jacobian noise: h = 1.5e-8*rho amplifies 1e-16 rounding

    def agree(a, b, tol):
        if shipped:
            return rel(a, b).max() < tol
        e = np.abs(a - b) / np.maximum(np.abs(b), 1e-9)     # a 1 x 1 patch solves exactly: costs of 1e-25 on both sides
        return (e < tol).mean() >= 0.99
    ok = r < 1e-7
    if lsnorm != capi.LSNORM_ZNCC:   # the reference leaves result[1] uninitialised for "zncc" (DepthProblemSolver.cpp:199-211)
        assert agree(pg["variance"][ok], po["variance"][ok], 1e-3)
    assert agree(pg["residual"][ok], po["residual"][ok], 1e-4)
    assert np.allclose(pg["p_cam"][ok], po["p_cam"][ok], rtol=1e-6, atol=1e-9)
    assert abs(evo - evg) <= 0.01 * evo


@pytest.mark.parametrize("lsnorm,patch", [(_ZN, (5, 5)), (_ZN, (11, 11)), (_L2, (5, 5)), (_TD, (5, 5)), (_TD, (11, 11))],
                         ids=["zncc-5x5", "zncc-11x11", "l2-5x5", "tdist-5x5", "tdist-11x11"])
def test_depth_solver_failed_warp_value(oracle_lib, product_lib, lsnorm, patch):
    """Seeds started at 6 x their matched inverse depth whose warp fails at the start and around it (checked with
    tests/indep_numpy.py): the residual is the constant failed-warp value (255 for l2, 2 / sqrt(N) for zncc, the weighted 255
    for Tdist), the Jacobian is zero and the solver stays put, so the reported cost is exactly N fv^2 -- at N != 105 this is
    what pins the kernels' failed-warp value."""
    import indep_numpy as ind
    s, o, g, so, sg, _, _ = _bm_pair(oracle_lib, product_lib, "hkust")
    o, g = make_backends("hkust", oracle_lib, product_lib, tweak=_tweak(lsnorm=lsnorm, patch_size_x=patch[0], patch_size_y=patch[1]))
    tl, tr = build_ts_pair(o, s)
    for be in (o, g):
        be.set_ts_pair(tl, tr, s["T_world_left"])
    Pl, Pr = (configs.rig_arrays("hkust")[k]["P"] for k in ("left", "right"))
    p = o.params
    norm = {_TD: "Tdist", _L2: "l2", _ZN: "zncc"}[lsnorm]
    Tlw = np.linalg.inv(s["T_world_left"])
    far = so.copy()
    far["inv_depth"] *= 6
    stuck = []
    for q in far:
        T = Tlw @ q["T_world_virtual"].reshape(4, 4)
        fails = []
        for x in q["inv_depth"] * np.array([1.0, 1 + 1.5e-8, 1.001, 0.999]):
            info = {}
            fv = ind.depth_residual(x, q["x_left"], T, Pl, Pr, tl, tr, patch[0], patch[1], p.td_nu, p.td_scale, norm, info)
            fails.append(info["failed"])
        if all(fails):
            stuck.append(q)
    stuck = np.array(stuck, dtype=capi.SEED_DTYPE)
    assert stuck.size > 100
    cost = float(fv @ fv)                                   # N fv^2 of the last failed evaluation
    po, _ = o.depth_solve(stuck)
    pg, _ = g.depth_solve(stuck)
    print(f"[lm failed warp {norm} {patch[0]}x{patch[1]}] {stuck.size} seeds, cost N fv^2 = {cost:.9g}; gpu costs {np.unique(pg['residual'])[:4]}")
    assert po.size == pg.size == stuck.size
    assert np.array_equal(po["inv_depth"], pg["inv_depth"]) and np.array_equal(np.sort(po["inv_depth"]), np.sort(stuck["inv_depth"]))
    assert np.all(np.abs(po["residual"] - cost) <= 1e-12 * cost) and np.all(np.abs(pg["residual"] - cost) <= 1e-12 * cost)


@pytest.mark.parametrize("kw", [dict(patch_size_x=16, patch_size_y=7), dict(patch_size_x=15, patch_size_y=8),
                                dict(patch_size_x=43, patch_size_y=3),                      # 129 pixels > kMaxPatch
                                dict(bm_step=2, invdepth_max_range=30.0, bm_max_disparity=400)],   # (400 - 3) / 2 + 1 = 199 coarse candidates
                         ids=["16x7", "15x8", "43x3", "step2-199cand"])
def test_create_refuses_unsupported_shapes(product_lib, kw):
    """Shapes no kernel serves are refused when the context is made, not mis-computed later: even patch sizes, more than 128
    patch pixels, and a coarse search of more than 192 candidates (the coarse cost map of bm_kernel) with step > 1."""
    l, r = configs.rig_calibs("hkust")
    with pytest.raises(capi.EsvoError) as e:
        capi.Backend(product_lib, l, r, _bm_case_params("hkust", kw, product_lib))
    assert e.value.code == -6                                          # ESVO_ERR_UNSUPPORTED
    if "bm_step" in kw:                                                # one candidate fewer is accepted
        capi.Backend(product_lib, l, r, _bm_case_params("hkust", dict(kw, bm_max_disparity=385), product_lib)).close()


@pytest.mark.parametrize("mode", ["radius0", "radius1", "naive"])
def test_fold_at_chosen_list_lengths(oracle_lib, product_lib, mode):
    """fuse_fold_kernel replays every pixel's contributions in sequence order, whatever the list length: lists of 1 .. 500
    contributions (util.FOLD_LENGTHS: both register networks, the three merged runs of 65 .. 192, the sort pool beyond, the
    255 bin of the length sort) on separate pixels, the points of all pixels interleaved, with depths and variances that make
    the surviving element depend on the replay order.  Device against the oracle and against tests/indep_fusion.py;
    esvo_fuse with radius 0 / 1 and esvo_naive_propagate (fuse_fold_kernel<true>)."""
    o, g = make_backends("hkust", oracle_lib, product_lib)
    Pl = configs.rig_arrays("hkust")["left"]["P"]
    pts, targets = fold_vector(Pl)
    radius = 1 if mode == "radius1" else 0
    nfs = []
    for be in (o, g):
        if mode == "naive":
            be.naive_propagate(pts, np.eye(4), True)
            nfs.append(0)
        else:
            nfs.append(be.fuse(pts, np.eye(4), radius, True))
    mo, mg = o.map_download(), g.map_download()
    grid, nfp = fold_replay(pts, Pl, o.W, o.H, radius, naive=mode == "naive")
    print(f"[fold {mode}] {pts.size} points on {len(targets)} pixels, map {mg.size} elements, fusions oracle {nfs[0]} gpu {nfs[1]}")
    assert mo.size == len(targets) * (9 if radius else 4)
    assert mode == "naive" or nfs[0] > 4000
    assert nfs[0] == nfs[1] == nfp
    assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"]), "element order differs"
    assert np.array_equal(mo["age"], mg["age"])
    maps_bit_identical(mo, mg, f"fold {mode}", p_cam_rtol=1e-9)      # p_cam: closed-form cam2World in the fold (DESIGN.md deviation 3)
    grid_vs_map(grid, mg, f"gpu {mode}")


def test_fusion_into_a_regularised_map(oracle_lib, product_lib):
    """DepthPoint::update_studentT takes its "new point" branch for a map point whose inverse depth is invalid
    (DepthPoint.cpp:181-187) -- reachable through the ABI: esvo_map_regularize marks rejected points with rho = -1, and a
    later esvo_fuse(reset_map = 0) fuses into them (ADVICE r1)."""
    s, o, g, so, sg, _, _ = _bm_pair(oracle_lib, product_lib, "hkust")
    po, _ = o.depth_solve(so)
    T0 = s["T_world_left"].copy()
    res = []
    for be in (o, g):
        be.fuse(po, T0, 0, True)
        be.map_regularize()
        m1 = be.map_download()
        nf = be.fuse(po[::2], T0, 0, False)            # second round into the regularised map, no reset
        res.append((m1, nf, be.map_download()))
    (a1, nfa, a2), (b1, nfb, b2) = res
    assert (a1["inv_depth"] <= -1e-6).sum() > 10, "the scenario must contain regularisation-rejected points"
    assert a1.size == b1.size and np.array_equal(a1["inv_depth"] > -1e-6, b1["inv_depth"] > -1e-6)
    assert nfa == nfb and a2.size == b2.size
    assert np.array_equal(a2["row"], b2["row"]) and np.array_equal(a2["col"], b2["col"]) and np.array_equal(a2["age"], b2["age"])
    v = a2["inv_depth"] > -1e-6
    assert np.array_equal(v, b2["inv_depth"] > -1e-6)
    maps_bit_identical(a2, b2, "fusion into a regularised map", p_cam_rtol=1e-9)
    # (With realistic variances a rejected point (rho = -1) is never within 2 sigma of a propagated one, so the second round
    #  goes through case 2.2 -- skip / replace -- for them; the "new point" branch itself needs a propagated rho near -1.)


@pytest.mark.parametrize("rig", ["hkust", "dsec"])
def test_cull_and_fusion_parity(oracle_lib, product_lib, rig):
    s, o, g, so, sg, _, _ = _bm_pair(oracle_lib, product_lib, rig)
    po, _ = o.depth_solve(so)
    p = o.params
    cost_thr = p.residual_vis_threshold ** 2 * p.patch_size_x * p.patch_size_y
    co = o.depth_cull(po, p.stdvar_vis_threshold, cost_thr, p.invdepth_min_range, p.invdepth_max_range)
    cg = g.depth_cull(po, p.stdvar_vis_threshold, cost_thr, p.invdepth_min_range, p.invdepth_max_range)
    assert co.size > 20 and co.size == cg.size and co.tobytes() == cg.tobytes()
    # fuse the same points three times from slightly different frame poses (exercises create / fuse / replace)
    T0 = s["T_world_left"].copy()
    for k, radius in enumerate((p.fusion_radius, p.fusion_radius, 1 - p.fusion_radius)):
        T = T0.copy(); T[0, 3] += 0.002 * k
        pts = co.copy()
        pts["T_world_cam"][:, 3] += 0.001 * k   # shift the observation poses a little
        nfo = o.fuse(pts, T0, radius, reset_map=(k == 0))
        nfg = g.fuse(pts, T0, radius, reset_map=(k == 0))
        assert nfo == nfg, f"round {k}: n_fusions {nfo} vs {nfg}"
    mo, mg = o.map_download(), g.map_download()
    assert mo.size == mg.size and mo.size > 0
    assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"]), "element order differs"
    maps_bit_identical(mo, mg, f"{rig} fusion", p_cam_rtol=1e-9)
    assert np.allclose(mo["p_cam"], mg["p_cam"], rtol=1e-9, atol=1e-12)
    o.map_clean(p.stdvar_vis_threshold ** 2, p.age_vis_threshold, p.invdepth_max_range, p.invdepth_min_range)
    g.map_clean(p.stdvar_vis_threshold ** 2, p.age_vis_threshold, p.invdepth_max_range, p.invdepth_min_range)
    o.map_regularize(); g.map_regularize()
    mo, mg = o.map_download(), g.map_download()
    assert mo.size == mg.size
    assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"])
    assert bits_equal(mo["inv_depth"], mg["inv_depth"]).all()


@pytest.mark.parametrize("rig,patch", [pytest.param("hkust", (15, 7), id="hkust"), pytest.param("dsec", (15, 7), id="dsec"),
                                        pytest.param("hkust", (5, 5), id="hkust-5x5"), pytest.param("hkust", (11, 11), id="hkust-11x11")])
def test_mapping_at_time_multi_frame(oracle_lib, product_lib, rig, patch):
    """Whole MappingAtTime over consecutive frames: window, fusion newest-first, clean, regularise.  Off the default patch
    shape the whole frame runs other BM and LM kernels, and the cull threshold (residual_vis_threshold^2 wx wy) changes."""
    def tw(p):
        p.max_num_fusion_frames = 3
        p.patch_size_x, p.patch_size_y = patch
    o = g = None
    for k, t_ts in enumerate((0.50, 0.55, 0.60, 0.65)):
        s = scenario(rig, n_seeds=800, t_ts=t_ts)
        if o is None:
            o, g = make_backends(rig, oracle_lib, product_lib, tweak=tw)
        tl, tr = build_ts_pair(o, s)
        o.ts_reset(0); o.ts_reset(1)
        sd = s["seeds"]
        for be in (o, g):
            be.set_ts_pair(tl, tr, s["T_world_left"])
        co = o.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        cg = g.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        print(rig, patch, k, co, cg)
        assert 200 < co["n_culled"] < co["n_solved"] and co["map_size"] > 500     # the cull removes points in every frame
        for key in ("n_events", "n_seeds", "n_solved", "n_culled", "bm_evals", "n_fusions", "map_size"):
            assert co[key] == cg[key], (k, key, co, cg)
        assert abs(co["lm_evals"] - cg["lm_evals"]) <= 0.01 * co["lm_evals"]
        mo, mg = o.map_download(), g.map_download()
        assert mo.size == mg.size
        assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"])
        r = rel(mg["inv_depth"], mo["inv_depth"])
        assert (r < 1e-4).mean() > 0.995 and np.median(r) < 1e-7


def test_initialization_from_sgm_disparity(oracle_lib, product_lib):
    """InitializationAtTime (esvo_Mapping.cpp:433-492): the node's own cv::StereoSGBM(0,48,11,968,3872,-1,0,11) on the TS pair,
    then edge mask AND disparity -> Gaussian DepthPoints -> naive_propagation; the following MappingAtTime frame fuses a
    window that contains the SGM vector."""
    import cv2
    s = scenario("hkust")
    o, g = make_backends("hkust", oracle_lib, product_lib)
    tl, tr = build_ts_pair(o, s)
    build_ts_pair(g, s)
    H, W = 260, 346
    sgbm = cv2.StereoSGBM_create(0, 48, 11, 8 * 11 * 11, 32 * 11 * 11, -1, 0, 11)
    disp = sgbm.compute(np.asarray(tl).reshape(H, W), np.asarray(tr).reshape(H, W))
    assert disp.dtype == np.int16 and (disp >= 0).mean() > 0.05
    sd = s["seeds"]
    T = s["T_world_left"]
    res = [be.init_from_disparity(disp, sd["x"], sd["y"], T, min_points=50) for be in (o, g)]
    assert res[0] == res[1] and res[0][1] and res[0][0] >= 50, res
    mo, mg = o.map_download(), g.map_download()
    assert mo.size == mg.size and mo.size > res[0][0]
    for f in ("row", "col", "age"):
        assert np.array_equal(mo[f], mg[f]), f
    for f in ("inv_depth", "variance", "residual", "x"):
        assert np.allclose(mo[f], mg[f], rtol=1e-13, atol=0), f
    assert np.allclose(mo["p_cam"], mg["p_cam"], rtol=1e-9, atol=1e-12)   # closed-form cam2World in the fold (DESIGN.md deviation 3)
    # the SGM vector itself (first vector of the window), element by element
    wo, wg = o.window_download(0), g.window_download(0)
    assert wo.size == wg.size == res[0][0]
    for f in wo.dtype.names:
        assert np.array_equal(wo[f], wg[f]), f                            # bit-exact incl. p_cam (same cofactor inverse)
    # too few points -> rejected, nothing pushed to the window
    r2 = [be.init_from_disparity(disp, sd["x"][:3], sd["y"][:3], T, min_points=50) for be in (o, g)]
    assert r2[0] == r2[1] and not r2[0][1]
    # re-initialise, then a regular mapping frame on top of the SGM vector
    for be in (o, g):
        be.mapping_reset()
        be.init_from_disparity(disp, sd["x"], sd["y"], T, min_points=50)
        be.set_ts_pair(tl, tr, T)
    co = o.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    cg = g.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
    assert co["n_seeds"] == cg["n_seeds"] and co["n_culled"] == cg["n_culled"] and co["map_size"] == cg["map_size"]
    assert co["n_fusions"] == cg["n_fusions"]
    mo, mg = o.map_download(), g.map_download()
    assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"])
    # The SGM points carry no Student-t scale / nu (the reference never initialises them: DepthPoint.cpp:7-35, UB there;
    # zero here and in the oracle), so pixels they fuse into turn NaN on both sides: compare NaN patterns, then values.
    a, b = mo["inv_depth"], mg["inv_depth"]
    assert np.array_equal(np.isnan(a), np.isnan(b))
    fin = ~np.isnan(a)
    r = rel(b[fin], a[fin])
    assert fin.sum() > 500 and (r < 1e-4).mean() > 0.995 and np.median(r) < 1e-7


def _track_run(c, oracle_lib, product_lib, max_iteration=None):
    """Case c of util.TRACK_CASES on the oracle and the device, identical inputs: [(pose, stats, permuted cloud, backend)]."""
    if max_iteration is not None:
        c = dict(c, it=max_iteration)
    tl, cloud, T_ref, T_prior = track_inputs(c, oracle_lib)
    res = []
    for lib in (oracle_lib, product_lib):
        be = track_backend(c, lib, product_lib)
        cl = cloud.copy()
        be.track_srand(1)
        assert be.track_reset(cl, T_ref, T_prior, tl) == 0
        T, st = be.track_solve(c["an"])
        res.append((T, st, cl, be))
    return res


# Pose bars (max abs over R and t / |t|), measured on one H100: analytic cases <= 7e-14, numerical <= 4.1e-7 (bar 1e-4).
# The one exception is the B = 6 line cloud, built so that two pairs of Jacobian columns are parallel to 1e-5 (smallest /
# largest singular value 1e-7): the device's reduction order is amplified by that condition number, 7.5e-7 after 20
# iterations with identical nfev / n_iter (DESIGN.md section 9).
TRACK_POSE_BAR = {True: 1e-8, False: 1e-4}
ILL_CONDITIONED_BAR = 1e-5
# The shipped hkust / dsec configurations: the solve must bring the translation from the prior's offset closer to the scene's
# true pose (measured: 5.4 -> 3.3 / 3.0 mm on hkust, 108 -> 24 / 18 mm on dsec, analytic / numerical).
TRACK_MOVES_TOWARDS_TRUTH = ("hkust-B500-huber50-k5-trans-an", "hkust-B500-huber50-k5-trans-num", "dsec-B300-huber50-k5-trans-an",
                             "dsec-B300-huber50-k5-trans-num")


def _pose_bar(c):
    return ILL_CONDITIONED_BAR if c["cloud"] == "line" else TRACK_POSE_BAR[c["an"]]


def _pose_dev(To, Tg):
    tn = max(np.linalg.norm(To[:3, 3]), 1e-3)
    return max(np.abs(To[:3, :3] - Tg[:3, :3]).max(), np.linalg.norm(To[:3, 3] - Tg[:3, 3]) / tn)


@pytest.mark.parametrize("cid", list(TRACK_CASES))
def test_tracking_negative_ts_and_sampling_bit_exact(oracle_lib, product_lib, cid):
    c = TRACK_CASES[cid]
    (_, _, co, o), (_, _, cg, g) = _track_run(c, oracle_lib, product_lib, max_iteration=1)
    for a, b in zip(o.track_get_negative_ts(), g.track_get_negative_ts()):
        assert np.array_equal(a, b)
    assert np.array_equal(co, cg), "rand()-driven partial shuffle differs"


@pytest.mark.parametrize("cid", list(TRACK_CASES))
def test_tracking_pose_parity(oracle_lib, product_lib, cid):
    """The whole RegProblemSolverLM solve of every case, device against oracle: n_points, nfev, n_iter exactly, the pose within
    TRACK_POSE_BAR.  Where the oracle trace shows a rejected trial, also after each k = 1 .. MAX_ITERATION on fresh contexts
    (MAX_ITERATION = k), so that equal totals cannot hide different trial sequences."""
    c = TRACK_CASES[cid]
    (To, so, co, o), (Tg, sg, cg, _) = _track_run(c, oracle_lib, product_lib)
    dev = _pose_dev(To, Tg)
    print(cid, so, sg, "pose deviation %.2e" % dev)
    assert so == sg
    assert np.array_equal(co, cg)
    assert dev < _pose_bar(c), dev
    tr = track_trace(o)
    if c["img"] == "const" or c["cloud"] == "off":
        # J == 0: status 4 at every iteration with x = 0.  addMotionUpdate(0) still passes R_ through the polar factor, which
        # moves it by rounding (6.7e-16 on one H100, differently on the two sides), so the pose is the prior to 1e-15, not bit for bit
        assert all(it["status"] == 4 for it in tr) and so["nfev"] == so["n_iter"] * (1 if c["an"] else 8)
        T_prior = track_inputs(c, oracle_lib)[3]
        assert dev < 1e-14 and np.abs(Tg - T_prior).max() < 1e-14 and np.abs(To - T_prior).max() < 1e-14
    if cid in TRACK_MOVES_TOWARDS_TRUTH:   # parity cannot see both sides standing still (or walking away) together
        Tw = scenario(c["rig"])["T_world_left"]
        T_prior = track_inputs(c, oracle_lib)[3]
        assert np.linalg.norm(Tg[:3, 3] - Tw[:3, 3]) < 0.7 * np.linalg.norm(T_prior[:3, 3] - Tw[:3, 3])
    if any(not q["accepted"] for it in tr for q in it["trials"]):
        for k in range(1, c["it"] + 1):
            (To, so, _, ok), (Tg, sg, _, _) = _track_run(c, oracle_lib, product_lib, max_iteration=k)
            assert so == sg, (k, so, sg)
            assert _pose_dev(To, Tg) < _pose_bar(c), (k, _pose_dev(To, Tg))


def test_tracking_device_ts_path_and_repeated_resets(oracle_lib, product_lib):
    """ts_left = NULL after a device ts_build gives the host-image result; two resets in a row without re-seeding keep the
    rand() streams (and so the shuffles and poses) equal on both sides."""
    c = TRACK_CASES["hkust-B500-huber50-k5-trans-an"]
    s = scenario("hkust")
    tl, cloud, T_ref, T_prior = track_inputs(c, oracle_lib)
    g = track_backend(c, product_lib, product_lib)
    tl_dev, _ = build_ts_pair(g, s)
    res = []
    for ts in (None, tl_dev):
        cl = cloud.copy()
        g.track_srand(1)
        assert g.track_reset(cl, T_ref, T_prior, ts) == 0
        res.append((g.track_solve(True), cl))
    assert np.array_equal(res[0][1], res[1][1]) and np.array_equal(res[0][0][0], res[1][0][0]) and res[0][0][1] == res[1][0][1]
    o = track_backend(c, oracle_lib, product_lib)
    o.track_srand(1); g.track_srand(1)
    for rep in range(2):
        out = []
        for be in (o, g):
            cl = cloud.copy()
            assert be.track_reset(cl, T_ref, T_prior, tl) == 0
            out.append((be.track_solve(True), cl))
        assert np.array_equal(out[0][1], out[1][1]), rep
        assert out[0][0][1] == out[1][0][1] and _pose_dev(out[0][0][0], out[1][0][0]) < 1e-8, rep


@pytest.mark.parametrize("kw", [dict(trk_batch_size=5), dict(trk_batch_size=1025), dict(trk_kernel_size=7)], ids=str)
def test_tracking_refuses_unsupported_parameters(oracle_lib, product_lib, kw):
    c = TRACK_CASES["hkust-B500-huber50-k5-trans-an"]
    tl, cloud, T_ref, T_prior = track_inputs(c, oracle_lib)
    l, r = configs.rig_calibs("hkust")
    p = track_params(c, product_lib)
    for k, v in kw.items():
        setattr(p, k, v)
    g = capi.Backend(product_lib, l, r, p)
    with pytest.raises(capi.EsvoError) as e:
        g.track_reset(cloud, T_ref, T_prior, tl)
    assert e.value.code == -6


def test_tracking_too_few_points(oracle_lib, product_lib):
    s = scenario("hkust")
    o, g = make_backends("hkust", oracle_lib, product_lib)
    tl, _ = build_ts_pair(o, s)
    cloud = np.zeros((10, 3), np.float32); cloud[:, 2] = 1
    for be in (o, g):
        assert be.track_reset(cloud.copy(), np.eye(4), np.eye(4), tl) == 1


@pytest.mark.parametrize("depth", [1, 3])
def test_pipelined_frames_match_oracle(oracle_lib, product_lib, depth):
    """Software-pipelined frames (esvo_set_pipeline_depth + esvo_results_begin/end) give the same per-frame
    maps and counters as the sequential oracle."""
    def tw(p):
        p.max_num_fusion_frames = 3
    o, g = make_backends("hkust", oracle_lib, product_lib, tweak=tw)
    g.set_pipeline_depth(depth)
    frames = [scenario("hkust", n_seeds=600, t_ts=t) for t in (0.50, 0.55, 0.60, 0.65, 0.70)]
    expected = []
    for s in frames:
        tl, tr = build_ts_pair(o, s)
        o.ts_reset(0); o.ts_reset(1)
        o.set_ts_pair(tl, tr, s["T_world_left"])
        sd = s["seeds"]
        c = o.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        expected.append((c, o.map_download(), tl, tr))
    tickets, got = [], []
    for k, s in enumerate(frames):
        if len(tickets) >= max(1, depth - 1):
            m, c = g.results_end(tickets.pop(0)); got.append((c, m.copy()))
        # device-resident TS hand-off: build the pair on the GPU from the raw events
        g.ts_reset(0); g.ts_reset(1)
        for cam, side in ((0, "left"), (1, "right")):
            e = s[side]
            g.stage_ts_events(cam, e["x"], e["y"], e["t"], e["p"])
            g.run_ts_build(cam, s["t_ts_ns"])
        T = np.ascontiguousarray(s["T_world_left"], np.float64)
        import ctypes as C
        g._call("set_ts_pair_dev", [C.POINTER(C.c_double)], T.ctypes.data_as(C.POINTER(C.c_double)))
        sd = s["seeds"]
        g.stage_mapping_inputs(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        g.run_mapping()
        tickets.append(g.results_begin())
    while tickets:
        m, c = g.results_end(tickets.pop(0)); got.append((c, m.copy()))
    assert len(got) == len(expected)
    for k, ((co, mo, _, _), (cg, mg)) in enumerate(zip(expected, got)):
        for key in ("n_events", "n_seeds", "n_solved", "n_culled", "bm_evals", "n_fusions", "map_size"):
            assert co[key] == cg[key], (k, key, co, cg)
        assert mo.size == mg.size
        assert np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"])
        r = rel(mg["inv_depth"], mo["inv_depth"])
        assert (r < 1e-4).mean() > 0.995 and np.median(r) < 1e-7


def test_time_surface_log_eviction(oracle_lib, product_lib):
    """Pushing more events than the resident log holds folds the oldest ones into the base grids; both the
    fast path (T newer than everything) and the general path (T inside the resident part) stay bit-exact."""
    o, g = make_backends("hkust", oracle_lib, product_lib)
    rng = np.random.default_rng(5)
    n_batch, n_batches = 1_500_000, 5            # 7.5 M events > 4 Mi resident
    t0 = 1_000_000_000
    for b in range(n_batches):
        x = rng.integers(0, 346, n_batch).astype(np.uint16); y = rng.integers(0, 260, n_batch).astype(np.uint16)
        # leave some pixels untouched after the first batch so that their value must come from the base grids
        if b > 0:
            x[x < 40] += 40
        t = (t0 + (b * n_batch + np.arange(n_batch)) * 40).astype(np.int64); p = rng.integers(0, 2, n_batch).astype(np.uint8)
        for be in (o, g):
            be.ts_push_events(0, x, y, t, p)
    t_end = int(t[-1])
    for T in (t_end + 1000, t_end - 200_000 * 40, t_end - 900_000 * 40):
        io, to = o.ts_build(0, T); ig, tg = g.ts_build(0, T)
        assert np.array_equal(io, ig), f"T={T}: {(io != ig).sum()} idx mismatches"
        assert np.array_equal(to, tg)


@pytest.mark.parametrize("rig", ["hkust", "dsec", "upenn"])
def test_product_rectification_tables_match_oracle(oracle_lib, product_lib, rig):
    """The library's own one-time host setup (maps, raw->rectified LUT, validity mask, baseline, disparity clip)
    against the oracle's, for plumb_bob and equidistant rigs."""
    l, r = configs.rig_calibs(rig)
    o = capi.Backend(oracle_lib, l, r, configs.params_for(rig, oracle_lib))
    g = capi.Backend(product_lib, l, r, configs.params_for(rig, product_lib))
    assert o.get_derived() == pytest.approx(g.get_derived(), rel=1e-14)
    for cam, cal in ((0, l), (1, r)):
        to, tg = o.get_rectify_tables(cam), g.get_rectify_tables(cam)
        th = capi.compute_rectify_tables(product_lib, cal)          # the context-free entry point returns what the ctx uses
        for a, b, c in zip(to, tg, th):
            assert np.array_equal(a, b) and np.array_equal(b, c)


def test_equidistant_rig_frame_parity(oracle_lib, product_lib):
    """One mapping frame on the reference's equidistant (upenn) rig, each side using ITS OWN rectification tables."""
    s = synth.make_stream("hkust", seed=6, n_seeds=800)      # event geometry from the hkust generator is fine: same sensor size
    l, r = configs.rig_calibs("upenn")
    o = capi.Backend(oracle_lib, l, r, configs.params_for("upenn", oracle_lib))
    g = capi.Backend(product_lib, l, r, configs.params_for("upenn", product_lib))
    res = []
    for be in (o, g):
        tl, tr = build_ts_pair(be, s)
        be.set_ts_pair(tl, tr, s["T_world_left"])
        sd = s["seeds"]
        c = be.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        res.append((tl, tr, c, be.map_download()))
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    for key in ("n_seeds", "n_solved", "n_culled", "bm_evals", "n_fusions", "map_size"):
        assert res[0][2][key] == res[1][2][key], (key, res[0][2], res[1][2])
    assert np.array_equal(res[0][3]["row"], res[1][3]["row"])
