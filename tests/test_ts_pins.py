"""Pins the oracle's time surface against re-derivations written from the reference sources only (tests/indep_numpy.py):
  * a2 FORWARD raster (TimeSurface.cpp:86-116: raster-order splat, clamp at 1 after every accumulation, no lower clamp, no remap)
  * a1 eventsCallback with out-of-order stamps (TimeSurface.cpp:403-425: every arrival queues events_.back())
  * every script of tests/util.py::TS_CASES (queue lengths, decay constants, stamp 0, events off the image, epoch stamps, ties,
    other image sizes, the hand-built FORWARD table, builds at and before the stamps the device folds out of its log), both modes
Index grid and published image bit for bit; no GPU.  The device runs the same scripts in tests/test_gpu_ts_parity.py, and
test_ts_cases_cover_every_branch asserts from the scripts themselves that they reach the branches of ts_push / ts_run_build."""
import numpy as np
import pytest

import indep_numpy as ind
from esvo_b200 import capi, configs
from util import (TS_CASES, TS_FWD_BLOCKS, TS_FWD_EXTRA, TS_LOG_CAP, TS_QLEN_PIX, TS_QLEN_T, TS_SIZES, scenario, ts_case_params, ts_case_script,
                  ts_cut, ts_effective, ts_handbuilt_lut, ts_host_model, ts_rig)

pytest.importorskip("cv2")


@pytest.mark.parametrize("rig,polarity,median", [("hkust", True, 1), ("hkust", True, 0), ("hkust", False, 1), ("hkust", False, 0),
                                                 ("dsec", True, 1), ("dsec", False, 0), ("upenn", True, 1), ("upenn", False, 0)])
def test_time_surface_forward_vs_numpy_and_cv2(oracle_lib, rig, polarity, median):
    """polarity = ignore_polarity.  With polarity in the value the sums fall below -1 (nothing clamps them there) and mono8 saturates."""
    s = scenario(rig, seed=2, n_seeds=100)
    l, r = configs.rig_calibs(rig)
    prm = configs.params_for(rig, oracle_lib)
    prm.time_surface_mode = 1; prm.ignore_polarity = 1 if polarity else 0; prm.median_blur_kernel_size = median
    o = capi.Backend(oracle_lib, l, r, prm)
    clamps, lowest = 0, 0.0
    for cam, side in ((0, "left"), (1, "right")):
        e = s[side]
        o.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
        lut = o.get_rectify_tables(cam)[2]
        n = e["t"].size
        for T in (s["t_ts_ns"], int(e["t"][n // 2]), int(e["t"][n // 5])):
            idx, ts = o.ts_build(cam, T)
            info = {}
            ref = ind.time_surface_forward(e, T, prm.decay_ms, o.W, o.H, polarity, median, lut, prm.max_event_queue_len, info)
            assert np.array_equal(idx, info["idx"]), (rig, cam, T)
            assert np.array_equal(ts, ref), (rig, cam, T, int((ts != ref).sum()))
            clamps += info["clamps"]; lowest = min(lowest, info["min_map"])
    print(f"[forward {rig} ignore_polarity={polarity} median={median}] clamps fired {clamps}, lowest sum {lowest:.3f}")
    assert clamps > 0
    assert polarity or lowest < -1


def _oracle(c, oracle_lib):
    l, r = configs.rig_calibs(ts_rig(c["size"]))
    prm = ts_case_params(c, oracle_lib)
    o = capi.Backend(oracle_lib, l, r, prm)
    if c["lut"]:
        o.set_rectify_tables(0, lut=c["lut"](o.W, o.H))
    return o, prm


def _rederive(o, prm, ev, T, info):
    m1, m2, lut, _ = o.get_rectify_tables(0)
    a = (ev, T, prm.decay_ms, o.W, o.H, bool(prm.ignore_polarity), prm.median_blur_kernel_size)
    if prm.time_surface_mode == 1:
        return ind.time_surface_forward(*a, lut, prm.max_event_queue_len, info)
    return ind.time_surface_backward(*a, m1, m2, prm.max_event_queue_len, info)[1]


def _run_script_on_oracle(c, oracle_lib):
    o, prm = _oracle(c, oracle_lib)
    ops = ts_case_script(c)
    eff = ts_effective(ops)
    seg = pushed = builds = 0
    stats = dict(clamps=0, min_map=0.0)
    for op in ops:
        if op[0] == "push":
            e = op[2]
            o.ts_push_events(0, e["x"], e["y"], e["t"], np.ones_like(e["p"]) if "nopol" in op[1] else e["p"])
            pushed += e["t"].size
        elif op[0] == "reset":
            o.ts_reset(0); seg += 1; pushed = 0
        elif op[0] in ("build", "refused"):                # what the device refuses the oracle and the re-derivation still agree on
            ev = ts_cut(eff[seg], 0, pushed)
            idx, ts = o.ts_build(0, op[1])
            info = {}
            ref = _rederive(o, prm, ev, op[1], info)
            assert np.array_equal(idx, info["idx"]), (c["id"], op[1], int((idx != info["idx"]).sum()))
            assert np.array_equal(ts, ref), (c["id"], op[1], int((ts != ref).sum()))
            stats["clamps"] += info.get("clamps", 0); stats["min_map"] = min(stats["min_map"], info.get("min_map", 0.0))
            builds += 1
    assert builds
    return stats


@pytest.mark.parametrize("cid", [k for k in TS_CASES if k != "evict-T-before-resident"])
def test_time_surface_scripts_vs_numpy(oracle_lib, cid):
    """Every build of every script: oracle against the re-derivation fed with what eventsCallback queues (arrival number as index)."""
    stats = _run_script_on_oracle(TS_CASES[cid], oracle_lib)
    if cid == "fwd-handbuilt":
        assert stats["clamps"] > 0 and stats["min_map"] < -1, stats


def test_time_surface_before_the_resident_log_vs_numpy(oracle_lib):
    """The oracle keeps the literal queues, so it answers any T; this makes it the judge of the builds the device accepts after
    folding its log, and shows that the ones the device refuses do have an answer it could no longer give."""
    _run_script_on_oracle(TS_CASES["evict-T-before-resident"], oracle_lib)


def test_events_callback_queue_hand_cases():
    q = lambda t: ind.events_callback_queue(dict(x=np.arange(len(t)), y=np.zeros(len(t), int), t=np.array(t), p=np.ones(len(t), int)))
    assert q([5, 3, 5, 4, 6, 6, 1])["x"].tolist() == [0, 0, 2, 2, 4, 5, 5]          # equal stamps: the later arrival is back()
    assert q([1, 2, 3])["x"].tolist() == [0, 1, 2]
    assert q([9, 1, 2, 3])["t"].tolist() == [9, 9, 9, 9]


def _contributions(W, H, ev):
    """Sources with an event whose table entry is accepted, counted per rectified pixel."""
    lut = ts_handbuilt_lut(W, H)
    src = np.zeros((H, W), bool)
    src[ev["y"], ev["x"]] = True
    cnt = np.zeros((H, W), int)
    for y, x in zip(*np.nonzero(src)):
        u, v = lut[y, x]
        if u >= 0 and v >= 0 and int(np.floor(u)) + 1 < W and int(np.floor(v)) + 1 < H:
            ui, vi = int(np.floor(u)), int(np.floor(v))
            for d in ((vi, ui), (vi, ui + 1), (vi + 1, ui), (vi + 1, ui + 1)):
                cnt[d] += 1
    return cnt, lut, src


def test_ts_cases_cover_every_branch():
    """From the scripts alone (push sizes and kinds, stamps against T, the table of the hand-built case): each named branch of
    ts_push / ts_run_build / the FORWARD fold is reached, so an edit of TS_CASES cannot quietly drop one."""
    seen, per_case = set(), {}
    for cid, c in TS_CASES.items():
        ops = ts_case_script(c)
        tags = ts_host_model(ops)
        per_case[cid] = (ops, tags)
        seen |= set().union(*tags)
    need = {"fast", "general", "general-launched-as-no-op", "empty-log", "T==host_max_t", "T==host_max_t+1", "T==oldest", "T==shared-stamp",
            "host", "nopol", "dev", "devnopol", "packet-one-copy", "packet-four-copies", "host-after-dev", "drain-refreshes-host",
            "order-violation-inside", "order-violation-across", "unordered", "scan-empty-carry", "scan-block-older-than-carry", "scan-tie",
            "scan-n1024", "scan-n1025", "scan-n2048", "scan-n1", "fold1", "fold2", "T<=folded", "T>folded", "T==oldest-resident"}
    assert need <= seen, sorted(need - seen)

    def tags_of(cid, kind=None):
        ops, tags = per_case[cid]
        return [t for o, t in zip(ops, tags) if kind is None or o[0] == kind]
    # kernels and parameters
    assert {TS_CASES[k]["prm"].get("median_blur_kernel_size") for k in ("bwd-median0", "bwd-median0-pol", "median2-refused")} == {0, 2}
    assert {c["prm"].get("decay_ms", 30.0) for c in TS_CASES.values()} >= {1.0, 30.0, 1000.0}
    assert {c["prm"].get("max_event_queue_len", 20) for c in TS_CASES.values()} >= {1, 2, 20, 64}
    # device pushes: the general kernels run as no-ops (no drain since), then do real work; after the drain the host decides again
    assert any("general-launched-as-no-op" in t for t in tags_of("dev-push", "build")) and any("general" in t for t in tags_of("dev-push", "build"))
    t = tags_of("dev-drain-then-build", "build")
    assert "fast" in t[0] and {"general", "T==host_max_t"} <= t[1] and "fast" in t[3] and "general-launched-as-no-op" in t[5]
    assert all("general" in t for t in tags_of("t-edges", "build") if "T==host_max_t" in t)
    assert sorted(o[2]["t"].size for o in per_case["packet-4095-4096"][0] if o[0] == "push")[:2] == [4095, 4096]
    # the scan: two or more whole blocks that lose to the carried event; a tie with it; pushes without polarity and from the device
    ops, tags = per_case["unord-carry-wins-blocks"]
    older = [o for o, t in zip(ops, tags) if "scan-block-older-than-carry" in t][0][2]["t"]
    carried = max(o[2]["t"].max() for o in ops[:2] if o[0] == "push")
    assert older.size >= 3 * 1024 and older.max() < carried
    assert any("scan-tie" in t for t in tags_of("unord-ties", "push"))
    assert any({"unordered", "nopol"} <= t for t in tags_of("unord-nopol")) and any({"unordered", "dev"} <= t for t in tags_of("unord-dev"))
    assert any({"unordered", "devnopol"} <= t for t in tags_of("unord-dev"))
    assert TS_CASES["unord-forward"]["prm"]["time_surface_mode"] == 1
    ops = [o[0] for o in per_case["unord-switched-on-late"][0]]
    assert ops.index("push") < ops.index("unordered_refused") < ops.index("reset") < ops.index("unordered")
    # the order flag: inside a push, across two pushes, a later ordered push before the reset, then a build after it
    for cid in ("order-flag", "order-flag-fwd"):
        ops, tags = per_case[cid]
        kinds = [("V" if t & {"order-violation-inside", "order-violation-across"} else "p") if o[0] == "push" else o[0][0] for o, t in zip(ops, tags)]
        assert "".join(kinds) == "pbVrrpVrprrpbbf", "".join(kinds)
    # queue lengths: exactly qlen - 1, qlen, qlen + 1 events that are not older than T, and an older one below them
    for q in (1, 2, 64):
        ev = ts_effective(per_case[f"qlen-{q}"][0])[0]
        for k, (px, py) in enumerate(TS_QLEN_PIX):
            on = (ev["x"] == px) & (ev["y"] == py)
            assert (ev["t"][on] >= TS_QLEN_T).sum() == q - 1 + k and (ev["t"][on] < TS_QLEN_T).sum() == 2
        assert ("build", TS_QLEN_T) in per_case[f"qlen-{q}"][0]
    # stamp 0, events off the image in front of events on it, epoch stamps closer than the spacing of doubles
    W, H = TS_SIZES["hkust"]
    ev = ts_effective(per_case["stamp0-offimage-epoch"][0])[0]
    off = (ev["x"] >= W) | (ev["y"] >= H)
    assert (ev["t"] == 0).sum() >= 2 and {W, 65535} <= set(ev["x"].tolist()) and H in ev["y"].tolist() and off[:6].any() and not off[-1]
    big = ev["t"][ev["t"] > 10 ** 18]
    assert big.size > 5000 and (np.diff(big) < 200).mean() > 0.9 and np.unique(big.astype(np.float64) * 1e-9).size < big.size // 2
    # sizes: partial tiles of the 32 x 8 raster kernels on both axes
    assert TS_SIZES["odd"][0] % 32 in (1, 31) and TS_SIZES["odd"][1] % 8 and TS_SIZES["small"][0] % 32 and {c["size"] for c in TS_CASES.values()} == set(TS_SIZES)
    # the hand-built table: destinations with more than 32, exactly 32 and 33 contributions; every rejection; polarity sums below -1
    ev = ts_effective(per_case["fwd-handbuilt"][0])[0]
    cnt, lut, src = _contributions(W, H, ev)
    assert cnt.max() == 100 and (cnt == 36).sum() == 4 and (cnt == 32).sum() == 2 and (cnt == 33).sum() == 2
    row0 = lut[0, :11]
    assert src[0, :11].all() and np.isnan(row0[0, 0]) and np.isnan(row0[7, 1]) and row0[1, 0] < 0 and row0[8, 1] < 0 and row0[2, 0] == W - 1 and \
        row0[3, 0] == W - 1.5 and row0[4, 0] == W and row0[5, 1] == H - 1 and row0[6, 1] == H - 1.5
    (x0, y0, w, h), _, pol = TS_FWD_BLOCKS[0]
    blk = (ev["x"] >= x0) & (ev["x"] < x0 + w) & (ev["y"] >= y0) & (ev["y"] < y0 + h)
    assert pol == 0 and not ev["p"][blk].any() and TS_CASES["fwd-handbuilt"]["prm"]["ignore_polarity"] == 0 and src[TS_FWD_EXTRA[0][1], TS_FWD_EXTRA[0][0]]
    # eviction: two folds, builds at the oldest resident stamp and one stamp before it, a push of more than half the log
    ops, tags = per_case["evict-T-before-resident"]
    b = [(o, t) for o, t in zip(ops, tags) if o[0] in ("build", "refused")]
    assert all(("T<=folded" in t) == (o[0] == "refused") for o, t in b)
    assert any("T==oldest-resident" in t and o[0] == "build" for o, t in b) and sum(o[0] == "refused" for o, _ in b) >= 3
    assert [o[1]["t"].size > TS_LOG_CAP // 2 for o in ops if o[0] == "push_refused"] == [True]
