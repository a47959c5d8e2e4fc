"""Seeded synthetic stereo event streams (SURVEY.md 8d): a 3-D scene of random line segments seen
by a moving rectified stereo rig; events are emitted in RAW (distorted) sensor coordinates whenever
a densely sampled edge point changes pixel.  Used by tests, bench.py and the golden-vector script.
numpy only -- generation is not part of the timed path.
"""
from __future__ import annotations

import numpy as np

from .configs import rig_arrays


def _rect_to_raw(cam, uv, equidistant=False):
    """Rectified pixel (sub-pixel) -> raw pixel: same math as initUndistortRectifyMap (plumb_bob, or with equidistant=True
    cv::fisheye::initUndistortRectifyMap)."""
    K, D, R, P = cam["K"], cam["D"], cam["R"], cam["P"]
    iR = np.linalg.inv(P[:, :3] @ R)
    h = np.concatenate([uv, np.ones((uv.shape[0], 1))], axis=1) @ iR.T
    x = h[:, 0] / h[:, 2]; y = h[:, 1] / h[:, 2]
    if equidistant:
        r = np.sqrt(x * x + y * y)
        th = np.arctan(r)
        th2 = th * th
        thd = th * (1 + th2 * (D[0] + th2 * (D[1] + th2 * (D[2] + th2 * D[3]))))
        s = np.where(r > 0, thd / np.maximum(r, 1e-300), 1.0)
        return np.stack([K[0, 0] * x * s + K[0, 2], K[1, 1] * y * s + K[1, 2]], axis=1)
    r2 = x * x + y * y
    kr = 1 + (D[1] * r2 + D[0]) * r2
    xd = x * kr + 2 * D[2] * x * y + D[3] * (r2 + 2 * x * x)
    yd = y * kr + D[2] * (r2 + 2 * y * y) + 2 * D[3] * x * y
    return np.stack([K[0, 0] * xd + K[0, 2], K[1, 1] * yd + K[1, 2]], axis=1)


def pose_at(t, amp=0.05, rot_deg=2.0, period=1.0):
    """Smooth trajectory T_world_left(t) (t in seconds)."""
    w = 2 * np.pi / period
    tr = amp * np.array([np.sin(w * t), 0.6 * np.sin(2 * w * t + 0.3), 0.4 * np.cos(w * t) - 0.4])
    a = np.deg2rad(rot_deg) * np.array([0.7 * np.sin(w * t + 0.5), np.sin(0.5 * w * t), 0.5 * np.sin(1.5 * w * t)])
    th = np.linalg.norm(a)
    Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    Rm = np.eye(3) if th < 1e-12 else np.eye(3) + np.sin(th) / th * Kx + (1 - np.cos(th)) / th ** 2 * (Kx @ Kx)
    T = np.eye(4)
    T[:3, :3] = Rm; T[:3, 3] = tr
    return T


def make_stream(rig="hkust", seed=2, t_ts=0.5, history_ms=60.0, n_segments=80, depth_range=None,
                n_seeds=5000, bm_window_ms=10.0, pose_dt_us=50.0, noise_frac=0.02, speed=1.0,
                sample_hz=1000.0, translation_scale=None, rig_model=False):
    """Returns a dict with left/right raw event arrays (sorted by time), the TS stamp, the seed
    events (newest first, as esvo_Mapping::dataTransferring gathers them, esvo_Mapping.cpp:562-575),
    the sampled virtual-view poses (:585-599) and the scene points.  translation_scale: the factor on the trajectory's
    translation (default 1 on hkust, 20 elsewhere); rig_model=True distorts with the rig's own model (equidistant on upenn)
    instead of plumb_bob everywhere."""
    cams = rig_arrays(rig)
    W, H = cams["width"], cams["height"]
    rng = np.random.default_rng(seed)
    if depth_range is None:
        depth_range = (0.5, 4.0) if rig == "hkust" else (4.0, 100.0)
    f = cams["left"]["P"][0, 0]; cx = cams["left"]["P"][0, 2]; cy = cams["left"]["P"][1, 2]
    # segments in the world frame (== left frame at the identity pose), sampled densely
    pts = []
    for _ in range(n_segments):
        z0 = rng.uniform(*depth_range); z1 = z0 * rng.uniform(0.8, 1.25)
        u0, v0 = rng.uniform(0.05 * W, 0.95 * W), rng.uniform(0.05 * H, 0.95 * H)
        ang = rng.uniform(0, 2 * np.pi); L = rng.uniform(0.15, 0.5) * W
        u1, v1 = u0 + L * np.cos(ang), v0 + L * np.sin(ang)
        n = int(2 * L) + 2
        s = np.linspace(0, 1, n)[:, None]
        a = np.array([(u0 - cx) * z0 / f, (v0 - cy) * z0 / f, z0]); b = np.array([(u1 - cx) * z1 / f, (v1 - cy) * z1 / f, z1])
        pts.append(a * (1 - s) + b * s)
    pts = np.concatenate(pts, axis=0)
    scale_t = (1.0 if rig == "hkust" else 20.0) if translation_scale is None else translation_scale  # translate more in the large-scale scene
    from .configs import RIGS
    equidistant = rig_model and RIGS[rig]["model"] == "equidistant"

    def project(t):
        T = pose_at(t * speed); T[:3, 3] *= scale_t
        Tinv = np.linalg.inv(T)
        pc = pts @ Tinv[:3, :3].T + Tinv[:3, 3]
        out = []
        for side in ("left", "right"):
            P = cams[side]["P"]
            hom = pc @ P[:, :3].T + P[:, 3]
            uv = hom[:, :2] / hom[:, 2:3]
            raw = _rect_to_raw(cams[side], uv, equidistant)
            ok = (pc[:, 2] > 0.1) & (raw[:, 0] >= 0) & (raw[:, 0] < W) & (raw[:, 1] >= 0) & (raw[:, 1] < H)
            out.append((np.floor(raw).astype(np.int64), ok))
        return out, T

    dt = 1.0 / sample_hz
    n_steps = int(round(history_ms * 1e-3 / dt))
    t0 = t_ts - n_steps * dt
    prev, _ = project(t0)
    ev = {"left": [], "right": []}
    for k in range(1, n_steps + 1):
        t = t0 + k * dt
        cur, _ = project(t)
        u_step = rng.uniform(0, 1, pts.shape[0]); pol_step = rng.integers(0, 2, pts.shape[0])
        for si, side in enumerate(("left", "right")):
            (pp, pok), (cp, cok) = prev[si], cur[si]
            moved = cok & pok & ((pp[:, 0] != cp[:, 0]) | (pp[:, 1] != cp[:, 1]))
            idx = np.nonzero(moved)[0]
            ts = (t - dt) + u_step[idx] * dt   # same sub-step phase / polarity in both cameras
            pol = pol_step[idx]
            ev[side].append(np.stack([cp[idx, 0], cp[idx, 1], (ts * 1e9).astype(np.int64), pol], axis=1))
        prev = cur
    out = {"W": W, "H": H, "rig": rig}
    t_ts_ns = int(round(t_ts * 1e9))
    for side in ("left", "right"):
        e = np.concatenate(ev[side], axis=0)
        nn = int(noise_frac * e.shape[0])
        noise = np.stack([rng.integers(0, W, nn), rng.integers(0, H, nn),
                          rng.integers(int(t0 * 1e9), t_ts_ns, nn), rng.integers(0, 2, nn)], axis=1)
        e = np.concatenate([e, noise], axis=0)
        e = e[e[:, 2] < t_ts_ns]
        e = e[np.argsort(e[:, 2], kind="stable")]
        out[side] = dict(x=e[:, 0].astype(np.uint16), y=e[:, 1].astype(np.uint16), t=e[:, 2].astype(np.int64),
                         p=e[:, 3].astype(np.uint8))
    out["t_ts_ns"] = t_ts_ns
    _, T_ts = project(t_ts)
    out["T_world_left"] = T_ts
    # seeds: newest first within the BM window
    L = out["left"]
    lo = np.searchsorted(L["t"], t_ts_ns - int(bm_window_ms * 1e6), side="left")
    sel = np.arange(L["t"].size - 1, lo - 1, -1)[:n_seeds]
    out["seeds"] = dict(x=L["x"][sel].copy(), y=L["y"][sel].copy(), t=L["t"][sel].copy())
    # virtual-view poses every pose_dt_us over the window (esvo_Mapping.cpp:585-599)
    tb = t_ts - bm_window_ms * 1e-3
    pt = np.arange(tb, t_ts + 0.5 * pose_dt_us * 1e-6, pose_dt_us * 1e-6)
    poses = []
    for t in pt:
        T = pose_at(t * speed); T[:3, 3] *= scale_t
        poses.append(T.ravel())
    out["pose_t"] = np.round(pt * 1e9).astype(np.int64)
    out["poses"] = np.array(poses)
    out["scene_points"] = pts
    return out
