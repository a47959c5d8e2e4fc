"""Device SGBM (esvo_sgbm_compute) against cv2.StereoSGBM, bit for bit, through the C ABI.

The arithmetic is also pinned on the host (tests/test_sgbm_core_host.py runs the very functions the kernels call).  The
device run happens in a subprocess with its own CUDA context (one-off start-up code, kept apart from the hot-path tests)."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (block size, number of disparities, uniqueness ratio, disp12MaxDiff): the sets tests/test_sgbm_core_host.py pins on the host
SGBM_SETS = [(11, 48, 11, -1), (5, 32, 0, 1000), (3, 16, 15, 2), (1, 16, 0, -1), (7, 64, 5, 1), (11, 128, 11, -1)]

CHILD = r'''
import sys, numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from esvo_b200 import capi, configs
from util import scenario, build_ts_pair
prod = capi.load_product()
l, r = configs.rig_calibs("hkust")
g = capi.Backend(prod, l, r, configs.params_for("hkust", prod), device=0)
s = scenario("hkust")
tl, tr = build_ts_pair(g, s)
tl = np.asarray(tl).reshape(260, 346); tr = np.asarray(tr).reshape(260, 346)
d_host = g.sgbm_compute(tl, tr)                      # host images
g.set_ts_pair(tl, tr, s["T_world_left"])
d_dev = g.sgbm_compute()                             # the observation pair that is on the device
d_small = g.sgbm_compute(tl, tr, 32, 5, None, None, 2, 0, 5)
sd = s["seeds"]
n, acc = g.init_from_disparity(d_host, sd["x"], sd["y"], s["T_world_left"], 50)
z = np.load(sys.argv[3])
sweep = {}
for pair in ("textured", "sparse"):
    for bs, nd, uq, d12 in z["sets"]:
        sweep[f"{pair}_{bs}_{nd}_{uq}_{d12}"] = g.sgbm_compute(z[pair + "_l"], z[pair + "_r"], int(nd), int(bs), None, None, int(d12), 0, int(uq))
l, r = configs.rig_calibs("dsec")
gd = capi.Backend(prod, l, r, configs.params_for("dsec", prod), device=0)
sweep["dsec"] = gd.sgbm_compute(z["dsec_l"], z["dsec_r"])
np.savez(sys.argv[2], tl=tl, tr=tr, d_host=d_host, d_dev=d_dev, d_small=d_small, n=n, acc=acc, **sweep)
'''


def _textured_pair(H, W, shift, seed):
    """Blurred noise seen with disparity `shift` in the upper half and `shift - shift // 2` in the lower half (the layout of
    test_sgbm_core_host.py's textured pair at full image size)."""
    import cv2
    rng = np.random.default_rng(seed)
    a = cv2.GaussianBlur(rng.integers(0, 256, (H, W + 2 * shift)).astype(np.uint8), (5, 5), 0)
    L, R = a[:, 0:W].copy(), a[:, shift:shift + W].copy()
    L[H // 2:, :] = a[H // 2:, shift // 2:shift // 2 + W]
    return L, R


def _sparse_pair(seed=5):
    """346 x 260 and sparse like a time surface: short bright strokes on zeros, disparity 12 (test_sgbm_core_host.py)."""
    import cv2
    rng = np.random.default_rng(seed)
    base = np.zeros((260, 400), np.uint8)
    for _ in range(120):
        y, x, n = rng.integers(5, 255), rng.integers(5, 360), rng.integers(5, 40)
        dy = rng.integers(-1, 2)
        for k in range(n):
            base[np.clip(y + dy * k // 3, 0, 259), x + k] = rng.integers(60, 255)
    base = cv2.GaussianBlur(base, (3, 3), 0)
    return base[:, 20:366].copy(), base[:, 32:378].copy()


@pytest.mark.gpu
def test_sgbm_device_matches_cv2(tmp_path):
    """The reference's parameters on the time-surface pair, and a sweep over block size, disparity count, uniqueness ratio
    and disp12MaxDiff on a textured and a sparse 346 x 260 pair, plus the reference's parameters on a 640 x 480 context."""
    import cv2
    out, inp = str(tmp_path / "sgbm_out.npz"), str(tmp_path / "sgbm_in.npz")
    tex_l, tex_r = _textured_pair(260, 346, 14, 3)
    sp_l, sp_r = _sparse_pair()
    ds_l, ds_r = _textured_pair(480, 640, 20, 4)
    np.savez(inp, sets=np.array(SGBM_SETS), textured_l=tex_l, textured_r=tex_r, sparse_l=sp_l, sparse_r=sp_r, dsec_l=ds_l, dsec_r=ds_r)
    p = subprocess.run([sys.executable, "-c", CHILD, ROOT, out, inp], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    z = np.load(out)
    ref = cv2.StereoSGBM_create(0, 48, 11, 8 * 121, 32 * 121, -1, 0, 11).compute(z["tl"], z["tr"])
    assert (ref >= 0).sum() > 20000
    assert np.array_equal(z["d_host"], ref)
    assert np.array_equal(z["d_dev"], ref)
    ref2 = cv2.StereoSGBM_create(0, 32, 5, 8 * 25, 32 * 25, 2, 0, 5).compute(z["tl"], z["tr"])
    assert np.array_equal(z["d_small"], ref2)
    assert bool(z["acc"]) and int(z["n"]) >= 50
    bad = []
    for pair, (L, R) in (("textured", (tex_l, tex_r)), ("sparse", (sp_l, sp_r))):
        for bs, nd, uq, d12 in SGBM_SETS:
            want = cv2.StereoSGBM_create(0, nd, bs, 8 * bs * bs, 32 * bs * bs, d12, 0, uq).compute(L, R)
            got = z[f"{pair}_{bs}_{nd}_{uq}_{d12}"]
            assert (want >= 0).sum() > 5000, (pair, bs, nd)
            print(f"[sgbm {pair} bs {bs} nd {nd} uq {uq} d12 {d12}] valid {(want >= 0).sum()}, differing pixels {(got != want).sum()}")
            if not np.array_equal(got, want):
                bad.append((pair, bs, nd, uq, d12, int((got != want).sum())))
    want = cv2.StereoSGBM_create(0, 48, 11, 8 * 121, 32 * 121, -1, 0, 11).compute(ds_l, ds_r)
    assert (want >= 0).sum() > 50000
    if not np.array_equal(z["dsec"], want):
        bad.append(("dsec 640x480", 11, 48, 11, -1, int((z["dsec"] != want).sum())))
    assert not bad, bad
