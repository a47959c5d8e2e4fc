"""Device against oracle on the map side, at the bit: esvo_fuse (fuse_stage_kernel, the ordered fold fold_apply), esvo_naive_propagate,
esvo_map_clean with thresholds on element values and both forms of esvo_map_regularize, over util.MAP_CASES and dense hand-built
maps.  Library and oracle both compute in f64 without contraction (-fmad=false, -ffp-contract=off) in the reference's order, so
every f64 field but p_cam (closed-form cam2World, DESIGN.md deviation 3) must carry the same bits; a NaN must be NaN on both
sides (x86 and the GPU produce different default NaN payloads)."""
import time

import numpy as np
import pytest

import indep_fusion as inf
from esvo_b200 import capi, configs, synth
from test_map_pins import REG_COUNTS, REG_RADII, dense_map
from util import MAP_CASES, bits_equal, build_ts_pair, make_backends, map_backends, map_round1, map_round2, maps_bit_identical, map_point, map_vec, rel

pytestmark = pytest.mark.gpu

W, H = 346, 260


def _pl():
    return configs.rig_arrays("hkust")["left"]["P"]


def _pick(v, q):
    """An element value at quantile q (a value the map really holds, so a threshold lands on it)."""
    v = np.sort(v[np.isfinite(v)])
    return float(v[int(q * (v.size - 1))]) if v.size else 0.0


def _clean_on_values(o, g, m, tag):
    """esvo_map_clean with each threshold on an element's value: age == age_thr, var == var_thr, rho == rmax, rho == rmin."""
    thr = (_pick(m["variance"], 0.5), _pick(m["age"].astype(np.float64), 0.5), _pick(m["inv_depth"], 0.8),
           _pick(m["inv_depth"], 0.2))
    for be in (o, g):
        be.map_clean(*thr)
    mo, mg = o.map_download(), g.map_download()
    maps_bit_identical(mo, mg, tag + f" clean {thr}")
    return mo.size


@pytest.mark.parametrize("cid", list(MAP_CASES))
def test_map_case_bit_identical(oracle_lib, product_lib, cid):
    """esvo_fuse round 1 (reset) and round 2 (no reset: the second-fold path, thresholds placed on the oracle's round-1 map),
    then esvo_map_clean on element values; esvo_naive_propagate of the same vector; all bit-identical to the oracle."""
    c = MAP_CASES[cid]
    Pl = _pl()
    t0 = time.time()
    o, g = map_backends(c, oracle_lib, product_lib)
    pts, T = map_round1(c, Pl)
    nf = [be.fuse(pts, T, c["radius"], True) for be in (o, g)]
    assert nf[0] == nf[1], (cid, nf)
    mo = o.map_download()
    maps_bit_identical(mo, g.map_download(), cid + " round 1")
    p2 = map_round2(c, mo, Pl)
    if p2 is not None:
        if c["r2"] == "regmap":
            for be in (o, g):
                be.map_regularize()
            maps_bit_identical(o.map_download(), g.map_download(), cid + " regularised")
        nf = [be.fuse(p2, T, c["radius"], False) for be in (o, g)]
        assert nf[0] == nf[1], (cid, "round 2", nf)
        maps_bit_identical(o.map_download(), g.map_download(), cid + " round 2")
    n_clean = _clean_on_values(o, g, o.map_download(), cid)
    for be in (o, g):
        be.naive_propagate(pts, T, True)
    maps_bit_identical(o.map_download(), g.map_download(), cid + " naive")
    print(f"[{cid}] {mo.size} elements, {nf[0]} fusions, {n_clean} after clean: bit-identical ({time.time() - t0:.2f} s)")


def test_map_clean_at_the_validity_threshold(oracle_lib, product_lib):
    """rho = -1e-6 and its neighbouring ulps (the edge case places them): the clean keeps exactly the elements above -1e-6."""
    c = MAP_CASES["tdist-r0-edge"]
    o, g = map_backends(c, oracle_lib, product_lib)
    pts, T = map_round1(c, _pl())
    for be in (o, g):
        be.fuse(pts, T, 0, True)
    m = o.map_download()
    near = np.abs(m["inv_depth"] + 1e-6) < 1e-20
    assert near.sum() == 12, m["inv_depth"][near]
    for be in (o, g):
        be.map_clean(np.inf, -np.inf, np.inf, -np.inf)
    mo, mg = o.map_download(), g.map_download()
    maps_bit_identical(mo, mg, "validity clean")
    assert (mo["inv_depth"] > -1e-6).all() and (np.abs(mo["inv_depth"] + 1e-6) < 1e-20).sum() == 4


def _reg_pair(oracle_lib, product_lib, norm, radius, mn, mc):
    def tw(p):
        p.lsnorm = capi.LSNORM_L2 if norm == "l2" else capi.LSNORM_TDIST
        p.reg_radius, p.reg_min_neighbours, p.reg_min_close_neighbours = radius, mn, mc
    return make_backends("hkust", oracle_lib, product_lib, tweak=tw)


def _reg_forms(o, g, pts, tag):
    """Oracle against both device forms: fuse(reset) + regularise (the warp list form), fuse(reset) + a second fold that
    touches no pixel + regularise (the image-wide thread form), and that form regularised twice in a row."""
    off = np.stack([map_point(_pl(), -5.0, 10.5, 0.5, s2=1e-4, exact=False)])      # outside the image: a fold, no pixel
    o.fuse(pts, np.eye(4), 0, True); o.map_regularize()
    mo = o.map_download()
    g.fuse(pts, np.eye(4), 0, True); g.map_regularize()
    ml = g.map_download()
    g.fuse(pts, np.eye(4), 0, True); g.fuse(off, np.eye(4), 0, False); g.map_regularize()
    mi = g.map_download()
    maps_bit_identical(mo, ml, tag + " list form")
    maps_bit_identical(mo, mi, tag + " image-wide form")
    o.map_regularize(); g.map_regularize()
    maps_bit_identical(o.map_download(), g.map_download(), tag + " twice")
    return mo


@pytest.mark.parametrize("norm", ["tdist", "l2"])
@pytest.mark.parametrize("radius", REG_RADII)
def test_regularisation_forms_bit_identical(oracle_lib, product_lib, norm, radius):
    """map_regularize_warp_kernel (one fold since the reset) and map_regularize_kernel<false> (any later fold) against the
    oracle at reg_radius 0 .. 20 (windows of 1 .. 1 681 pixels: 1, 2, 4, 8 and 53 chunks of 32 lanes) and min counts
    0 / 0, 8 / 8, 32 / 32; at radius 2 and 5 also min_nb / min_close at count - 1 and count of chosen pixels (the tests
    are strict: the pixel flips between kept and rejected)."""
    Pl = _pl()
    pts = dense_map(Pl, norm)
    t0 = time.time()
    for mn, mc in (REG_COUNTS if radius < 20 else REG_COUNTS[1:2]):
        o, g = _reg_pair(oracle_lib, product_lib, norm, radius, mn, mc)
        mo = _reg_forms(o, g, pts, f"{norm} r={radius} {mn}/{mc}")
        assert mo.size > 1000 and (mo["inv_depth"] == -1.0).any()
    if radius in (2, 5):
        grid = inf.Grid(H, W)
        inf.fuse_vector(grid, map_vec(pts), np.eye(4), Pl, W, H, 0, norm="l2" if norm == "l2" else "Tdist")
        flips = 0
        for (row, col) in ((radius, radius), (radius + 7, radius + 3), (H - 1 - radius, W - 1 - radius)):
            e = grid.cell.get((row, col))
            if e is None or not e.valid():
                continue
            nbs = grid.neighbourhood(row, col, radius)
            close = [q for q in nbs if abs(e.rho - q.rho) < 2.0 * np.sqrt(e.var) or abs(e.rho - q.rho) < 2.0 * np.sqrt(q.var)]
            kept = []
            for mn, mc in ((len(nbs) - 1, 0), (len(nbs), 0), (0, len(close) - 1), (0, len(close))):
                o, g = _reg_pair(oracle_lib, product_lib, norm, radius, mn, mc)
                mo = _reg_forms(o, g, pts, f"{norm} r={radius} {mn}/{mc} at ({row}, {col})")
                k = int(np.nonzero((mo["row"] == row) & (mo["col"] == col))[0][0])
                kept.append(mo["inv_depth"][k] != -1.0)
            assert kept[0] and not kept[1] and kept[2] and not kept[3], (row, col, len(nbs), len(close), kept)
            flips += 1
        assert flips >= 2
    print(f"[reg {norm} r={radius}] bit-identical in both forms ({time.time() - t0:.2f} s)")


def test_create_refuses_negative_reg_radius(product_lib):
    """A negative radius is an empty neighbourhood loop for the reference but not for the warp form's (2r+1)^2 window:
    esvo_create refuses it; radius 0 (the pixel itself) is accepted."""
    l, r = configs.rig_calibs("hkust")
    p = configs.params_for("hkust", product_lib)
    p.reg_radius = -1
    with pytest.raises(capi.EsvoError) as ei:
        capi.Backend(product_lib, l, r, p)
    assert ei.value.code == -6
    p.reg_radius = 0
    capi.Backend(product_lib, l, r, p).close()


# ---- MappingAtTime with fusion windows past the 32 vectors of one staging launch (fuse_window) and past the 64 of the
# order array in capi_map.cu, and with FUSION_CONST_POINTS eviction on the device.  Few seeds per frame keep the oracle
# side short (the frames are synthesised once per rig and shared by the runs).
WIN_SEEDS = 150
_FRAMES = {}


def _frames(rig, n):
    fr = _FRAMES.setdefault(rig, [])
    while len(fr) < n:
        fr.append(synth.make_stream(rig, seed=2, n_seeds=WIN_SEEDS, t_ts=0.3 + 0.012 * len(fr)))
    return fr[:n]


WINDOW_RUNS = {
    "hkust-33": ("hkust", dict(max_num_fusion_frames=33), 36),          # two staging launches: 32 + 1 vectors
    "hkust-40": ("hkust", dict(max_num_fusion_frames=40), 43),          # the upenn value: 32 + 8
    "hkust-65": ("hkust", dict(max_num_fusion_frames=65), 68),          # three launches and the order copy past 64
    "hkust-points": ("hkust", dict(fusion_strategy=capi.FUSION_CONST_POINTS, max_num_fusion_points=250, max_num_fusion_frames=4), 14),
    "upenn-yaml": ("upenn", dict(), 43),                                # the shipped upenn yaml (maxNumFusionFrames = 40)
}


def _lm_bar(a, b):
    if a.size:
        r = rel(b, a)
        assert (r < 1e-4).mean() >= 0.995 and np.median(r) < 1e-7, (r.max(), np.median(r))


def _same_vector(vo, vg, tag):
    assert vo.size == vg.size, (tag, vo.size, vg.size)
    for f in ("row", "col", "age"):
        assert np.array_equal(vo[f], vg[f]), (tag, f)
    assert bits_equal(vo["x"], vg["x"]).all() and bits_equal(vo["T_world_cam"], vg["T_world_cam"]).all(), tag
    _lm_bar(vo["inv_depth"], vg["inv_depth"])


@pytest.mark.parametrize("run", list(WINDOW_RUNS))
def test_mapping_window_past_one_staging_launch(oracle_lib, product_lib, run):
    """MappingAtTime frame after frame until the window is full and then evicts: per frame the counters (lm_evals within
    1 %, as in test_mapping_at_time_multi_frame), the map order and the window length exact, inverse depth at the LM bar
    (>= 99.5 % within 1e-4, median < 1e-7), and the oldest and newest window vectors (esvo_window_download) equal to the
    oracle's: rows / cols, ages, x and poses exact, inverse depth at the LM bar."""
    rig, kw, n = WINDOW_RUNS[run]

    def tw(p):
        for k, v in kw.items():
            setattr(p, k, v)
    frames = _frames(rig, n)
    o, g = make_backends(rig, oracle_lib, product_lib, tweak=tw)
    prm = o.params
    t_oracle, t0 = 0.0, time.time()
    sizes, full = [], 0
    for k, s in enumerate(frames):
        tl, tr = build_ts_pair(o, s)
        o.ts_reset(0); o.ts_reset(1)
        sd = s["seeds"]
        for be in (o, g):
            be.set_ts_pair(tl, tr, s["T_world_left"])
        t1 = time.time()
        co = o.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        t_oracle += time.time() - t1
        cg = g.mapping_at_time(sd["x"], sd["y"], sd["t"], s["pose_t"], s["poses"])
        for key in ("n_events", "n_seeds", "n_solved", "n_culled", "bm_evals", "n_fusions", "map_size"):
            assert co[key] == cg[key], (run, k, key, co, cg)
        assert abs(co["lm_evals"] - cg["lm_evals"]) <= 0.01 * co["lm_evals"]
        mo, mg = o.map_download(), g.map_download()
        assert mo.size == mg.size and np.array_equal(mo["row"], mg["row"]) and np.array_equal(mo["col"], mg["col"]), (run, k)
        _lm_bar(mo["inv_depth"], mg["inv_depth"])
        # the window: the reference's eviction rule applied to the culled vector sizes (esvo_Mapping.cpp:342-368)
        sizes.append(co["n_culled"])
        if prm.fusion_strategy == capi.FUSION_CONST_POINTS:
            while sum(sizes) > 1.5 * prm.max_num_fusion_points:
                sizes.pop(0); full += 1
        elif len(sizes) > prm.max_num_fusion_frames:
            sizes.pop(0); full += 1
        nw = len(sizes)
        for be in (o, g):
            with pytest.raises(capi.EsvoError):
                be.window_download(nw)
        for idx in (0, nw - 1):
            _same_vector(o.window_download(idx), g.window_download(idx), f"{run} frame {k} window[{idx}]")
    assert full >= 3, (run, full)                  # the window filled and then evicted for several frames
    print(f"[window {run}] {n} frames, window {len(sizes)} vectors, {full} evictions; oracle mapping {t_oracle:.2f} s, "
          f"test {time.time() - t0:.2f} s")
