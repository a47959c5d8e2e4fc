"""Event windows read from the time-surface log (include/esvo_b200.h: esvo_events_window_dev, esvo_events_lower_bound_dev and the
_selected_dev frames) against their host forms byte for byte: the walk of frontend::selectCloseEvents / selectSGMEvents
(tests/indep_numpy.py) over the node's deque, createDenoisingMask + extractDenoisedEvents (cv2.medianBlur), and
tools::EventBuffer_lower_bound; refusals where the resident log cannot answer; the mapping frames on a selection against the
host-array calls on the same events; and the closed loop with Denoising off against its restatement."""
import numpy as np
import pytest

import event_window_cases as ewc
from esvo_b200 import capi

pytestmark = pytest.mark.gpu

ERR_STATE, ERR_UNSUPPORTED = -5, -6


def _backend(product_lib):
    from esvo_b200 import configs
    l, r = configs.rig_calibs("hkust")
    return capi.Backend(product_lib, l, r, configs.params_for("hkust", product_lib))


def _push(g, case):
    off = 0
    for b in case["batches"]:
        sl = slice(off, off + b)
        g.ts_push_events(0, case["x"][sl], case["y"][sl], case["t"][sl], np.ones(b, np.uint8))
        off += b
    assert off == case["t"].size


@pytest.mark.parametrize("name", list(ewc.cases()))
def test_windows_and_bounds_match_host_form(product_lib, name):
    case = ewc.cases()[name]
    secs = ewc.stream_secs(case)
    g = _backend(product_lib)
    _push(g, case)
    answered = refused = 0
    for q in case["queries"]:
        exp = ewc.expect(case, q, secs)
        if q[0] == "window":
            _, front, tb, te, budget, denoise, max_keep = q
            rc, n = g.events_window_dev(0, front, tb, te, budget, denoise, max_keep, ok=(0, ERR_UNSUPPORTED))
            if exp is None:
                assert rc == ERR_UNSUPPORTED, (name, q)
                refused += 1
                continue
            assert rc == 0, (name, q)
            sel, _ = exp
            x, y, t = g.events_selected_dev()
            assert n == sel.size == x.size, (name, q, n, sel.size)
            assert x.tobytes() == case["x"][sel].tobytes() and y.tobytes() == case["y"][sel].tobytes(), (name, q)
            assert t.tobytes() == case["t"][sel].tobytes(), (name, q)
            answered += 1
        else:
            _, front, stamps = q
            for s, e in zip(stamps, exp):           # one at a time: each bound is answered exactly or refused on its own
                rc, idx = g.events_lower_bound_dev(0, front, [s], ok=(0, ERR_UNSUPPORTED))
                if rc == 0:
                    assert idx[0] == e, (name, q, s, idx[0], e)
                    answered += 1
                else:
                    assert not ewc.lower_bound_answerable(case, front, s, secs), (name, q, s)
                    refused += 1
            known = np.array([ewc.lower_bound_answerable(case, front, s, secs) for s in stamps])
            for k in range(0, len(stamps), 64):      # at most 64 stamps per call: the determined bounds are written, the others -1
                rc, idx = g.events_lower_bound_dev(0, front, stamps[k: k + 64], ok=(0, ERR_UNSUPPORTED))
                kn = known[k: k + 64]
                assert rc == (0 if kn.all() else ERR_UNSUPPORTED), (name, q)
                assert np.array_equal(idx, np.where(kn, exp[k: k + 64], -1)), (name, q)
    print(f"{name}: {answered} answered, {refused} refused")
    assert answered > 0 and (refused > 0) == (name == "evicted")


def test_window_host_forms_agree(product_lib):
    """The selections the shim's host form makes (indep_numpy.select_close_events / select_sgm_events) equal the walk of the
    case table at the windows dataTransferring uses."""
    import indep_numpy as ind
    case = ewc.cases()["epoch"]
    secs = ewc.stream_secs(case)
    for q in case["queries"][:60]:
        if q[0] != "window":
            continue
        _, front, tb, te, budget, _, _ = q
        host = ind.select_close_events(case["t"][front:], te, 0.001, budget) if budget == 1000 else \
            ind.select_sgm_events(case["t"][front:], te, 0.001, budget - 1)
        assert np.array_equal(host, ewc.walk(secs[front:], tb, te, budget))


def test_refusals(product_lib):
    """Unordered input, stamps pushed out of order, depth > 1, a front past the log, t_begin > t_end."""
    rng = np.random.default_rng(3)
    x, y = rng.integers(0, 346, 100).astype(np.uint16), rng.integers(0, 260, 100).astype(np.uint16)
    t = np.arange(100, dtype=np.int64) * 1000 + 10**6
    g = _backend(product_lib)
    g.ts_set_unordered_input(0, True)
    g.ts_push_events(0, x, y, t, np.ones(100, np.uint8))
    assert g.events_window_dev(0, 0, 0, 10**9, 100, 1, 100, ok=(ERR_UNSUPPORTED,))[0] == ERR_UNSUPPORTED
    assert g.events_lower_bound_dev(0, 0, [10**6], ok=(ERR_UNSUPPORTED,))[0] == ERR_UNSUPPORTED
    g = _backend(product_lib)
    g.ts_push_events(0, x, y, t[::-1].copy(), np.ones(100, np.uint8))
    assert g.events_window_dev(0, 0, 0, 10**9, 100, 0, 100, ok=(ERR_UNSUPPORTED,))[0] == ERR_UNSUPPORTED
    assert g.events_lower_bound_dev(0, 0, [10**6], ok=(ERR_UNSUPPORTED,))[0] == ERR_UNSUPPORTED
    g = _backend(product_lib)
    g.ts_push_events(0, x, y, t, np.ones(100, np.uint8))
    assert g.events_window_dev(0, 101, 0, 10**9, 100, 0, 100, ok=(-1,))[0] == -1
    assert g.events_window_dev(0, 0, 10**9, 10**6, 100, 0, 100, ok=(-1,))[0] == -1
    with pytest.raises(capi.EsvoError) as e:            # no selection yet
        g.mapping_at_time_selected_dev(np.zeros(0, np.int64), np.zeros((0, 16)))
    assert e.value.code == ERR_STATE
    g.set_pipeline_depth(2)
    assert g.events_window_dev(0, 0, 0, 10**9, 100, 0, 100, ok=(ERR_STATE,))[0] == ERR_STATE
    assert g.events_lower_bound_dev(0, 0, [10**6], ok=(ERR_STATE,))[0] == ERR_STATE


def _frame_pair(product_lib):
    """Two contexts with the same time surfaces built and the same observation set (smoke()'s stream)."""
    from esvo_b200 import synth
    s = synth.make_stream("hkust", seed=7, n_seeds=400, n_segments=60)
    out = []
    for _ in range(2):
        g = _backend(product_lib)
        for cam, side in ((0, "left"), (1, "right")):
            e = s[side]
            g.ts_push_events(cam, e["x"], e["y"], e["t"], e["p"])
        g.ts_build(0, s["t_ts_ns"]); g.ts_build(1, s["t_ts_ns"])
        g.set_ts_pair(None, None, s["T_world_left"])
        out.append(g)
    return s, out


@pytest.mark.parametrize("denoise", [1, 0])
def test_mapping_on_selection_equals_host_arrays(product_lib, denoise):
    s, (g, h) = _frame_pair(product_lib)
    e = s["left"]
    te = int(s["t_ts_ns"])
    tb = ewc.t_begin_for(te, 0.01)
    pen = 2000
    rc, n = g.events_window_dev(0, 0, tb, te, pen, denoise, pen)
    walked = ewc.walk(ewc.to_sec(e["t"]), tb, te, pen)
    x, y = e["x"][walked], e["y"][walked]
    sel = walked[ewc.extract(x, y, ewc.mask_of(x, y), pen)] if denoise else walked
    assert n == sel.size and walked.size == pen - 1, (n, sel.size, walked.size)   # t_end is newer than every event
    x, y, t = g.events_selected_dev()
    assert x.tobytes() == e["x"][sel].tobytes() and y.tobytes() == e["y"][sel].tobytes() and t.tobytes() == e["t"][sel].tobytes()
    print(f"denoise {denoise}: {n} of {walked.size} walked events selected")
    cg = g.mapping_at_time_selected_dev(s["pose_t"], s["poses"])
    ch = h.mapping_at_time(e["x"][sel], e["y"][sel], e["t"][sel], s["pose_t"], s["poses"])
    assert cg == ch and cg["n_events"] == n, (cg, ch)
    assert g.map_download().tobytes() == h.map_download().tobytes()


def test_init_on_selection_equals_host_arrays(product_lib):
    s, (g, h) = _frame_pair(product_lib)
    e = s["left"]
    te = int(s["t_ts_ns"])
    tb = ewc.t_begin_for(te, 0.002)
    pen = 1000
    _, n = g.events_window_dev(0, 0, tb, te, pen + 1, 0, pen + 1)
    sel = ewc.walk(ewc.to_sec(e["t"]), tb, te, pen + 1)
    assert n == sel.size > 0
    disp = g.sgbm_compute(None, None)
    assert np.array_equal(disp, h.sgbm_compute(None, None))
    for thr in (1, 10**6):                         # accepted, and refused for too few points
        rg = g.init_from_disparity_selected_dev(disp, s["T_world_left"], thr)
        rh = h.init_from_disparity(disp, e["x"][sel], e["y"][sel], s["T_world_left"], thr)
        assert rg == rh and rg[0] > 0, (rg, rh)
        assert g.map_download().tobytes() == h.map_download().tobytes()


def test_system_loop_denoising_off_matches_restatement(product_lib, tmp_path):
    """The closed loop on the "mapping" scene with Denoising off: the C++ system (device windows) against the restatement on the
    product (host windows), identical records and final-map bytes."""
    import indep_system as isy
    import test_system_loop as tsl
    s = tsl._stream("mapping")
    t0, n = tsl._ticks(s)
    (sh_ticks, sh_maps, sh_map, stopped, _, _, _), _ = tsl._run_shim(tmp_path, s, t0, n, ((2, 0.0),))
    assert stopped == 0 and sh_ticks.size == n
    g = _backend(product_lib)
    pr_ticks, pr_maps, pr_map, _, err = isy.run_system(g, lambda l, r: g.sgbm_compute(l, r), s["left"], s["right"], t0, tsl.DT_NS, n,
                                                       denoising=False)
    assert err is None
    diff = tsl._first_difference(sh_ticks, sh_maps, pr_ticks, pr_maps, 0.0, True)
    assert diff is None, f"first difference at tick {diff[0]}: {diff[1]}"
    assert sh_map.tobytes() == pr_map.tobytes()
    assert (sh_maps["ran"] == 2).sum() > 0 and sh_maps[sh_maps["ran"] == 2]["ctr"][:, 0].max() > 0


def test_tracker_count_device_form_equals_host_form(product_lib, tmp_path):
    """esvo_Tracking::curDataTransferring's numEventsSinceLastObs_ from its own deque and from the log (examples/tracker_count_dump.cpp)
    at every tick of an epoch-stamped stream, with two reset()s: the device form's deque starts at the push index of the reset."""
    import os
    import struct
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build = os.path.join(root, "esvo_b200", "_build")
    exe = str(tmp_path / "tracker_count_dump")
    subprocess.check_call(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), os.path.join(root, "examples", "tracker_count_dump.cpp"),
                           "-L" + build, "-lesvo_b200", "-Wl,-rpath," + build, "-o", exe])
    rng = np.random.default_rng(8)
    n = 200_000
    t = ewc.EPOCH + np.cumsum(rng.integers(0, 200, n)).astype(np.int64)
    x = rng.integers(0, 346, n).astype(np.uint16); y = rng.integers(0, 260, n).astype(np.uint16)
    ticks = np.linspace(t[0] + 1, t[-1] + 1, 120).astype(np.int64)
    resets = np.zeros(ticks.size, np.int32); resets[[30, 31, 77]] = 1
    with open(tmp_path / "in.bin", "wb") as f:
        f.write(struct.pack("<i", ticks.size)); f.write(ticks.tobytes()); f.write(resets.tobytes())
        f.write(struct.pack("<i", n)); f.write(x.tobytes()); f.write(y.tobytes()); f.write(t.tobytes())
    p = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    c = np.fromfile(tmp_path / "out.bin", np.uint64).reshape(-1, 2)
    assert c.shape[0] == ticks.size and (c[:, 0] > 0).sum() > 100
    assert np.array_equal(c[:, 0], c[:, 1]), np.nonzero(c[:, 0] != c[:, 1])[0]
