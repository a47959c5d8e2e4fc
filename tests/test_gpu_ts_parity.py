"""Time-surface parity beyond the shipped configuration: every script of tests/util.py::TS_CASES run on the CUDA path and on the
CPU oracle alike, index grid and published image equal at every build, every refusal asserted with its error code.  The oracle
side of the same scripts is pinned against an independent re-derivation in tests/test_ts_pins.py, which also asserts that the
scripts reach each branch of ts_push / ts_run_build (esvo_b200/csrc/ts.cu)."""
import ctypes as C

import numpy as np
import pytest

from esvo_b200 import capi, configs
from util import TS_CASES, TS_UNSUPPORTED, ts_case_params, ts_case_script, ts_rig

pytestmark = pytest.mark.gpu

u16, i64, u8 = C.POINTER(C.c_uint16), C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
PUSH_ARGS = [C.c_int, u16, u16, i64, u8, C.c_size_t]


def _backends(c, oracle_lib, product_lib):
    l, r = configs.rig_calibs(ts_rig(c["size"]))
    o = capi.Backend(oracle_lib, l, r, ts_case_params(c, oracle_lib))
    g = capi.Backend(product_lib, l, r, ts_case_params(c, product_lib))
    for cam in (0, 1):                       # the product runs on its own tables; the oracle gets the same ones
        m1, m2, lut, mask = g.get_rectify_tables(cam)
        if c["lut"]:
            lut = c["lut"](g.W, g.H)
            g.set_rectify_tables(cam, lut=lut)
        o.set_rectify_tables(cam, m1, m2, lut, mask)
    return o, g


def _push_product(g, cam, how, e, keep):
    import torch
    n = e["t"].size
    x, y, t, p = (np.ascontiguousarray(e[k]) for k in ("x", "y", "t", "p"))
    if how == "host":
        g.ts_push_events(cam, x, y, t, p)
    elif how == "nopol":
        g._call("ts_push_events", PUSH_ARGS, cam, x.ctypes.data_as(u16), y.ctypes.data_as(u16), t.ctypes.data_as(i64), None, n)
    elif how in ("dev", "devnopol"):
        d = [torch.from_numpy(a.view(np.uint8).copy()).cuda() for a in (x, y, t, p)]
        torch.cuda.synchronize()             # the copies ran on torch's stream, the push runs on the context's
        keep.append(d)                       # the push is asynchronous: the arrays live until the next build has synchronised
        ptr = lambda k, ty: C.cast(d[k].data_ptr(), ty)
        g._call("ts_push_events_dev", PUSH_ARGS, cam, ptr(0, u16), ptr(1, u16), ptr(2, i64), None if how == "devnopol" else ptr(3, u8), n)
    else:                                    # one host buffer t | x | y | p, handed over as four (packet) or three (packetnopol) arrays
        buf = np.zeros(13 * n + 16, np.uint8)
        bt = buf[0:8 * n].view(np.int64); bx = buf[8 * n:10 * n].view(np.uint16); by = buf[10 * n:12 * n].view(np.uint16); bp = buf[12 * n:13 * n]
        bt[:] = t; bx[:] = x; by[:] = y; bp[:] = p
        g._call("ts_push_events", PUSH_ARGS, cam, bx.ctypes.data_as(u16), by.ctypes.data_as(u16), bt.ctypes.data_as(i64),
                bp.ctypes.data_as(u8) if how == "packet" else None, n)


def _refused(code, f, *a):
    with pytest.raises(capi.EsvoError) as e:
        f(*a)
    assert e.value.code == code, e.value
    return str(e.value)


@pytest.mark.parametrize("cid", list(TS_CASES))
def test_time_surface_case(oracle_lib, product_lib, cid):
    c = TS_CASES[cid]
    ops = ts_case_script(c)
    o, g = _backends(c, oracle_lib, product_lib)
    l, r = configs.rig_calibs(ts_rig(c["size"]))
    builds = 0
    for cam in c["cams"]:
        keep, last = [], None
        for k, op in enumerate(ops):
            tag = (cid, cam, k, op[0], op[1] if len(op) > 1 and not isinstance(op[1], dict) else "")
            if op[0] == "push":
                e = op[2]
                o.ts_push_events(cam, e["x"], e["y"], e["t"], np.ones_like(e["p"]) if "nopol" in op[1] else e["p"])
                _push_product(g, cam, op[1], e, keep)
            elif op[0] == "build":
                io, to = o.ts_build(cam, op[1])
                ig, tg = g.ts_build(cam, op[1])
                keep.clear()
                assert np.array_equal(io, ig), (tag, f"{(io != ig).sum()} index mismatches")
                assert np.array_equal(to, tg), (tag, f"{(to != tg).sum()} image mismatches")
                last = (ig, tg)
                builds += 1
            elif op[0] == "refused":
                msg = _refused(op[2], g.ts_build, cam, op[1])
                keep.clear()
                if cid.startswith("evict"):                   # the message names the oldest T that can still be answered
                    oldest = int(msg.rsplit(" ", 1)[1])
                    assert op[1] < oldest
                    io, to = o.ts_build(cam, oldest); ig, tg = g.ts_build(cam, oldest)
                    assert np.array_equal(io, ig) and np.array_equal(to, tg), (tag, oldest)
            elif op[0] == "push_refused":
                _refused(op[2], _push_product, g, cam, "host", op[1], keep)
            elif op[0] == "sync":
                g.sync()
            elif op[0] == "reset":
                o.ts_reset(cam); g.ts_reset(cam)
            elif op[0] == "unordered":
                g.ts_set_unordered_input(cam, op[1])
            elif op[0] == "unordered_refused":
                _refused(TS_UNSUPPORTED, g.ts_set_unordered_input, cam, 1)
            elif op[0] == "fresh":
                f = capi.Backend(product_lib, l, r, ts_case_params(c, product_lib))
                _push_product(f, cam, "host", op[1], keep)
                i2, t2 = f.ts_build(cam, op[2])
                assert np.array_equal(i2, last[0]) and np.array_equal(t2, last[1]), tag
                assert i2.max() < op[1]["t"].size              # the index grid restarted at 0
                f.close()
            else:
                raise KeyError(op[0])
        g.sync()                                               # a refusal leaves the context usable
    assert builds or cid == "median2-refused"
    o.close(); g.close()
