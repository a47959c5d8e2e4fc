"""Independent restatement of the multi-view stereo system (include/esvo_b200/esvo_mvstereo_system.hpp), written from the
REFERENCE source esvo_core/src/esvo_MVStereo.cpp: MappingLoop (:179-237), MappingAtTime (:239-520), dataTransferring
(:552-668), stampedPoseCallback (:670-706), getPoseAt (:709-744), eventsCallback / timeSurfaceCallback (:746-838), reset
(:840-880), publishMappingResults / publishPointCloud (:960-1039), vEMP2vDP (:1072-1094), eventSlicingForEM (:1096-1125),
with the tf buffer of tests/indep_system.py.  Drives any capi.Backend: the per-pixel stages run through the C ABI,
everything node-level is plain Python here.  TEST INFRASTRUCTURE: clarity over speed.
"""
import numpy as np

import indep_numpy as ind
import indep_system as isy

# the rpg ground truth is the pose of the marker; the camera is T_world_marker * T_marker_cam (:731-735)
T_MARKER_CAM = np.array([[5.363262328777285e-01, -1.748374625145743e-02, -8.438296573030597e-01, -7.009849865398374e-02],
                         [8.433577587813513e-01, -2.821937531845164e-02, 5.366109927684415e-01, 1.881333563905305e-02],
                         [-3.319431623758162e-02, -9.994488408486204e-01, -3.897382049768972e-04, -6.966829200678797e-02],
                         [0, 0, 0, 1]])
MAX_NUM_EVENT_INVOLVED = 10000                  # :639
# examples/mvstereo_system.cpp's per-frame record
FRAME_DTYPE = np.dtype([("tick", "<i4"), ("t", "<i8"), ("gated", "<i4"), ("transferred", "<i4"), ("ran", "<i4"), ("ok", "<i4"),
                        ("published", "<i4"), ("stamp", "<i8"), ("T_kf", "<f8", (16,)), ("n_left", "<u8"), ("n_right", "<u8"),
                        ("n_sgm", "<u8"), ("n_window", "<u8"), ("n_close", "<u8"), ("n_st", "<u8"), ("n_matches", "<u8"),
                        ("cloud_points", "<u8"), ("resets", "<u8"), ("ms", "<f8")], align=False)
COUNT_KEYS = ("n_left", "n_right", "n_sgm", "n_window", "n_close", "n_st", "n_matches", "cloud_points", "resets")


def secs(t):
    """ros::Time::toSec() of every stamp (sec + 1e-9 * nsec, the same double operations as ind.ros_to_sec)."""
    t = np.asarray(t, np.int64)
    s, n = np.divmod(t, 1000000000)
    return s.astype(np.float64) + 1e-9 * n.astype(np.float64)


def inconsistent(t_new, t_old):
    """max_time_diff_before_reset_s = 0.5 (:675,752,800)."""
    dt = ind.ros_to_sec(t_new) - ind.ros_to_sec(t_old)
    return dt < 0 or abs(dt) >= 0.5


class Queue:
    """EventQueue: x, y, t, p arrays in queue order (stable by stamp: the insertion sort moves only strictly later events)."""

    def __init__(self):
        self.clear()

    def clear(self):
        self.x = np.zeros(0, np.uint16); self.y = np.zeros(0, np.uint16); self.t = np.zeros(0, np.int64); self.p = np.zeros(0, np.uint8)
        self.s = np.zeros(0)

    def add(self, e):
        x = np.concatenate([self.x, e["x"]]); y = np.concatenate([self.y, e["y"]])
        t = np.concatenate([self.t, np.asarray(e["t"], np.int64)]); p = np.concatenate([self.p, e["p"]])
        o = np.argsort(t, kind="stable")
        keep = o[max(0, o.size - 3000000):]          # clearEventQueue (:782-790)
        self.x, self.y, self.t, self.p = x[keep], y[keep], t[keep], p[keep]
        self.s = secs(self.t)

    def lower_bound(self, t_ns):
        """tools::EventBuffer_lower_bound: compares toSec() doubles."""
        return int(np.searchsorted(self.s, ind.ros_to_sec(t_ns), side="left"))

    def take(self, idx):
        idx = np.asarray(idx, np.int64)
        return dict(x=self.x[idx], y=self.y[idx], t=self.t[idx], p=self.p[idx])


def no_events():
    return dict(x=np.zeros(0, np.uint16), y=np.zeros(0, np.uint16), t=np.zeros(0, np.int64), p=np.zeros(0, np.uint8))


class Node:
    """The node's host state: queues, TS history, tf, the reset rules and dataTransferring.  Callbacks return True when a
    reset ran; the caller then drops the map (see System)."""

    def __init__(self, W, H, mode, pen=500, ts_len=100, em_num=3000, half=0.001, denoising=False, marker=False):
        self.W, self.H, self.mode = W, H, mode
        self.pen, self.ts_len, self.em_num, self.half, self.denoising, self.marker = pen, ts_len, em_num, half, denoising, marker
        self.left, self.right = Queue(), Queue()
        self.ts = {}                                  # TS_history_: stamp -> (left, right)
        self.tf = isy.PoseBuffer()
        self.tf_latest = 0
        self.resets = 0
        self.obs = None                               # TS_obs_: (stamp, T) or None
        self.em_left = self.em_right = self.sgm = self.window = self.close = no_events()
        self.t_low = self.t_up = 0
        self.st_t, self.st_T = np.zeros(0, np.int64), np.zeros((0, 16))

    def reset(self):                                  # :840-880 (the map part is the owner's)
        self.left.clear(); self.right.clear(); self.ts.clear(); self.tf = isy.PoseBuffer()
        self.resets += 1

    def events(self, e, left):                        # :746-780
        if e["t"].size == 0:
            return False
        q = self.left if left else self.right
        r = q.t.size > 0 and inconsistent(int(e["t"][0]), int(q.t[-1]))
        if r:
            self.reset()
        q.add(e)
        return r

    def time_surface(self, t, tl, tr):                # :792-838
        r = bool(self.ts) and inconsistent(t, max(self.ts))
        if r:
            self.reset()
        self.ts.setdefault(t, (tl, tr))               # emplace: an existing stamp keeps its images
        while len(self.ts) > self.ts_len:
            del self.ts[min(self.ts)]
        return r

    def pose(self, t, T):                             # :670-706
        if self.tf.t:                                 # getLatestCommonTime writes only on success
            self.tf_latest = self.tf.t[-1]
        r = ind.ros_to_sec(self.tf_latest) != 0 and inconsistent(t, self.tf_latest)
        if r:
            self.reset()
        self.tf.set_transform(t, T)
        return r

    def pose_at(self, t):                             # :709-744
        T = self.tf.lookup(t)
        if T is None or not self.marker:
            return T
        out = np.zeros((4, 4))
        for r in range(4):
            for c in range(4):
                out[r, c] = T[r, 0] * T_MARKER_CAM[0, c] + T[r, 1] * T_MARKER_CAM[1, c] + T[r, 2] * T_MARKER_CAM[2, c] + T[r, 3] * T_MARKER_CAM[3, c]
        return out

    def clear_selection(self):
        """Start of a pass: no observation, no selection (a pass without an observation leaves nothing behind)."""
        self.obs = None
        self.em_left = self.em_right = self.sgm = self.window = self.close = no_events()
        self.st_t, self.st_T = np.zeros(0, np.int64), np.zeros((0, 16))

    def data_transferring(self):                      # :552-668
        self.clear_selection()
        if len(self.ts) <= 10:
            return False
        stamps = sorted(self.ts)
        for t in stamps[-2::-1]:                      # from the newest but one back to the oldest
            T = self.pose_at(t)
            if T is not None:
                self.obs = (t, T)
                break
        if self.obs is None:
            return False
        t_obs = self.obs[0]
        if self.mode in (0, 2):                       # :579-609
            self.t_low, self.t_up = stamps[0], stamps[-1]
            bounds = []
            for q in (self.left, self.right):
                lo, up = q.lower_bound(self.t_low), q.lower_bound(self.t_up) - 1
                if lo >= up:                          # one event (lo == up) -- or none, where the reference walks off
                    return False
                bounds.append((lo, min(up, lo + self.em_num + 1)))    # `<=`: EM_numEventMatching + 1 events
            (a, b), (c, d) = bounds
            self.em_left, self.em_right = self.left.take(np.arange(a, b)), self.right.take(np.arange(c, d))
        if self.mode == 4:                            # :612-625
            self.sgm = self.left.take(ind.select_sgm_events(self.left.t, t_obs, self.half, self.pen))
        if self.mode in (1, 3):                       # :628-666
            self.window = self.left.take(ind.select_close_events(self.left.t, t_obs, self.half, MAX_NUM_EVENT_INVOLVED))
            st, sp = [], []
            for s in ind.sample_pose_stamps(t_obs, self.half):
                T = self.pose_at(int(s))
                if T is not None:
                    st.append(int(s)); sp.append(T.ravel())
            self.st_t, self.st_T = np.array(st, np.int64), np.array(sp).reshape(-1, 16)
        return True

    def denoise(self):                                # :385-405
        w = self.window
        if self.denoising:
            import cv2
            img = np.zeros((self.H, self.W), np.uint8)
            img[w["y"].astype(int), w["x"].astype(int)] = 255
            mask = cv2.medianBlur(img, 3)
            keep = np.nonzero(mask[w["y"].astype(int), w["x"].astype(int)] == 255)[0][: self.pen]
        else:
            keep = np.arange(min(w["t"].size, self.pen))
        self.close = {k: v[keep] for k, v in w.items()}

    def prepare(self):
        """The host part of one MappingLoop pass (:196-225): (gated, transferred, MappingAtTime due)."""
        if len(self.ts) < 10:
            self.clear_selection()
            return False, False, False
        ok = self.data_transferring()
        if self.obs is None:                          # TS_obs_ empty: skip (the return value is not looked at)
            return True, ok, False
        if self.mode in (1, 3):
            self.denoise()
        return True, ok, True


class System:
    """esvo_MVStereoSystem on one Backend: the node above plus MappingAtTime (:239-520) and the publishers."""

    def __init__(self, be, sgbm, cfg, Pl00, t0_ns, dt_ns):
        """sgbm(tl, tr) -> CV_16S disparity (cv::StereoSGBM(0, 48, 11, 968, 3872, -1, 0, 11)); Pl00: P(0, 0) of the left camera."""
        p = be.params
        self.be, self.sgbm, self.cfg, self.Pl00, self.t0, self.dt = be, sgbm, cfg, Pl00, t0_ns, dt_ns
        self.node = Node(be.W, be.H, cfg["MVStereoMode"], cfg["PROCESS_EVENT_NUM"], cfg["TS_HISTORY_LENGTH"], cfg["EM_NUM_EVENT_MATCHING"],
                         cfg["BM_half_slice_thickness"], cfg["Denoising"], cfg["dvs_frame_id"] == "marker")
        self.every = max(1, int(np.floor(1e9 / (cfg["mapping_rate_hz"] * dt_ns) + 0.5)))
        self.window = []                              # dqvDepthPoints_
        self.fresh = True                             # the current DepthFrame holds no map
        self.max_frames, self.max_points = p.max_num_fusion_frames, p.max_num_fusion_points

    def drop_map(self, reset):
        if reset:
            self.window = []; self.fresh = True
            self.be.mapping_reset()

    def get_map(self):
        from esvo_b200 import capi
        return self.be.map_download() if not self.fresh else np.zeros(0, capi.DEPTH_POINT_DTYPE)

    def _accumulate_naive(self, vdp, T):             # :281-286, :357-361, :423-427
        self.window.append(vdp)
        del self.window[:-self.max_frames]
        for q, v in enumerate(reversed(self.window)):
            self.be.naive_propagate(v, T, q == 0)
        self.fresh = False

    def mapping_at_time(self, tl, tr, T):
        """Returns (ok, number of matches)."""
        be, n, p, mode = self.be, self.node, self.be.params, self.node.mode
        self.fresh = True                             # a new DepthFrame (:247-251)
        vemp = None
        if mode in (0, 2):                            # :257-306
            counts, med = ind.event_slicing_for_em(n.em_left["t"], n.t_low, n.t_up, self.cfg["EM_Slice_Thickness"]) \
                if n.em_left["t"].size else (np.zeros(0, np.int32), np.zeros(0, np.int64))
            poses = []
            for m in med:
                Tm = n.pose_at(int(m))
                poses.append(np.zeros(16) if Tm is None else Tm.ravel())
            if counts.size == 0:
                return False, 0
            be.set_ts_pair(tl, tr, T)
            vemp, _ = be.em_match(n.em_left, n.em_right, counts, np.array(poses).reshape(-1, 16), time_thr=self.cfg["EM_Time_THRESHOLD"],
                                  epi_thr=self.cfg["EM_EPIPOLAR_THRESHOLD"], ncc_thr=self.cfg["EM_TS_NCC_THRESHOLD"],
                                  patch=(p.patch_size_x, p.patch_size_y), num_thread=4)
            if vemp.size == 0:
                return False, 0
            if mode == 0:
                self._accumulate_naive(be.seeds_to_points(vemp), T)
                return True, vemp.size
        if mode == 4:                                 # :311-376
            be.set_ts_pair(tl, tr, T)
            disp = self.sgbm(tl, tr)
            self._accumulate_naive(sgm_points(be, n.sgm, disp, T, self.Pl00), T)
            return True, 0
        if mode in (1, 3):                            # :383-435
            be.set_ts_pair(tl, tr, T)
            c = n.close
            vemp, _ = be.bm_match(c["x"], c["y"], c["t"], n.st_t, n.st_T)
            if mode == 1:
                self._accumulate_naive(be.seeds_to_points(vemp), T)
                return True, vemp.size
        if vemp.size:                                 # :445-507
            be.set_ts_pair(tl, tr, T)
            vdp, _ = be.depth_solve(vemp)
        else:
            from esvo_b200 import capi
            vdp = np.zeros(0, capi.DEPTH_POINT_DTYPE)
        cost_thr = p.residual_vis_threshold ** 2 * p.patch_size_x * p.patch_size_y
        vdp = be.depth_cull(vdp, p.stdvar_vis_threshold, cost_thr, p.invdepth_min_range, p.invdepth_max_range)
        self.window.append(vdp)
        if p.fusion_strategy == 1:                    # CONST_POINTS
            while sum(v.size for v in self.window) > 1.5 * self.max_points:
                self.window.pop(0)
        else:
            del self.window[:-self.max_frames]
        for q, v in enumerate(reversed(self.window)):
            be.fuse(v, T, p.fusion_radius, q == 0)
        self.fresh = False
        be.map_clean(p.stdvar_vis_threshold ** 2, p.age_vis_threshold, p.invdepth_max_range, p.invdepth_min_range)
        if p.regularization:
            be.map_regularize()
        return True, vemp.size

    def run(self, left, right, pose_t, poses, n_ticks, keep_maps=False):
        """The fixed schedule (DESIGN.md section 5).  Returns (FRAME_DTYPE records, final map, per-frame maps or None)."""
        be, n = self.be, self.node
        done = [0, 0]; done_pose = 0
        frames, maps = [], []
        for k in range(n_ticks):
            t = self.t0 + k * self.dt
            batch = []
            for cam, e in enumerate((left, right)):
                hi = int(np.searchsorted(e["t"], t, side="left"))
                b = {key: e[key][done[cam]:hi] for key in ("x", "y", "t", "p")}
                if hi > done[cam]:
                    be.ts_push_events(cam, b["x"], b["y"], b["t"], b["p"])
                done[cam] = hi
                batch.append(b)
            _, tl = be.ts_build(0, t, want_idx=False)
            _, tr = be.ts_build(1, t, want_idx=False)
            self.drop_map(n.events(batch[0], True)); self.drop_map(n.events(batch[1], False))
            self.drop_map(n.time_surface(t, tl, tr))
            if k % self.every:
                continue
            while done_pose < len(pose_t) and pose_t[done_pose] <= t:
                self.drop_map(n.pose(int(pose_t[done_pose]), poses[done_pose]))
                done_pose += 1
            rec = np.zeros((), FRAME_DTYPE)
            rec["tick"], rec["t"] = k, t
            gated, ok, due = n.prepare()
            rec["gated"], rec["transferred"] = gated, ok
            if due:
                t_obs, T = n.obs
                ltl, ltr = n.ts[t_obs]
                rec["ran"], rec["stamp"], rec["T_kf"] = 1, t_obs, T.ravel()
                rec["n_left"], rec["n_right"] = n.em_left["t"].size, n.em_right["t"].size
                rec["n_sgm"], rec["n_window"], rec["n_close"], rec["n_st"] = n.sgm["t"].size, n.window["t"].size, n.close["t"].size, n.st_t.size
                done_ok, rec["n_matches"] = self.mapping_at_time(ltl, ltr, T)
                rec["ok"] = done_ok
                if done_ok:
                    m = self.get_map()
                    rec["cloud_points"] = m.size
                    rec["published"] = int(m.size > 0)
                    if keep_maps:
                        maps.append((k, m))
            rec["resets"] = n.resets
            frames.append(rec)
        return np.array(frames, FRAME_DTYPE), self.get_map(), (maps if keep_maps else None)


def sgm_points(be, ev, disp16, T, Pl00, num_disparities=48):
    """The PURE_SEMI_GLOBAL_MATCHING branch between the SGM call and the accumulation (:320-352): createEdgeMask(undistorted
    events, radius 0), x < numDisparities and disp < 0 skipped, var 0, residual 0, DepthPoint(x, y) taking (x, y) as (row, col)."""
    from esvo_b200 import capi
    lut = be.get_rectify_tables(0)[2]
    c = np.floor(lut[ev["y"].astype(int), ev["x"].astype(int)]).astype(np.int64)
    inside = (c[:, 0] >= 0) & (c[:, 0] < be.W) & (c[:, 1] >= 0) & (c[:, 1] < be.H)
    c = c[inside]
    disp = disp16[c[:, 1], c[:, 0]] / 16.0
    keep = (c[:, 0] >= num_disparities) & (disp >= 0)
    c, disp = c[keep], disp[keep]
    seeds = np.zeros(c.shape[0], capi.SEED_DTYPE)
    seeds["x_left"] = c.astype(np.float64)
    seeds["inv_depth"] = disp / (Pl00 * be.get_derived()["baseline"])
    seeds["T_world_virtual"] = np.asarray(T, float).ravel()
    pts = be.seeds_to_points(seeds)
    pts["row"], pts["col"] = c[:, 0], c[:, 1]
    return pts


# ---- the files of examples/mvstereo_system.cpp and examples/mvstereo_node_dump.cpp ----
def write_scenario(path, lcal, rcal, params, t0_ns, dt_ns, n_ticks, cfg, left, right, pose_t, poses, profile=False):
    import ctypes as C
    import struct
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", C.sizeof(lcal), C.sizeof(params)))
        f.write(bytes(lcal)); f.write(bytes(rcal)); f.write(bytes(params))
        f.write(struct.pack("<qqid", t0_ns, dt_ns, n_ticks, float(cfg["mapping_rate_hz"])))
        f.write(struct.pack("<7i", cfg["MVStereoMode"], cfg["PROCESS_EVENT_NUM"], cfg["TS_HISTORY_LENGTH"], cfg["EM_NUM_EVENT_MATCHING"],
                            int(cfg["Denoising"]), int(cfg["dvs_frame_id"] == "marker"), int(profile)))
        f.write(struct.pack("<5d", cfg["BM_half_slice_thickness"], cfg["EM_Slice_Thickness"], cfg["EM_Time_THRESHOLD"],
                            cfg["EM_EPIPOLAR_THRESHOLD"], cfg["EM_TS_NCC_THRESHOLD"]))
        for e in (left, right):
            f.write(struct.pack("<i", e["x"].size))
            for a, dt in ((e["x"], np.uint16), (e["y"], np.uint16), (e["t"], np.int64), (e["p"], np.uint8)):
                f.write(np.ascontiguousarray(a, dt).tobytes())
        f.write(struct.pack("<i", len(pose_t)))
        f.write(np.asarray(pose_t, np.int64).tobytes()); f.write(np.ascontiguousarray(poses, np.float64).reshape(-1, 16).tobytes())


def parse_result(path):
    """-> (frames, map, stopped, wall_ms, stage_ms, stage_launches)."""
    from esvo_b200 import capi
    raw = open(path, "rb").read()
    n_f, n_map, stopped = np.frombuffer(raw, np.int32, 3)
    off = 12
    fr = np.frombuffer(raw, FRAME_DTYPE, n_f, off).copy(); off += n_f * FRAME_DTYPE.itemsize
    m = np.frombuffer(raw, capi.DEPTH_POINT_DTYPE, n_map, off).copy(); off += n_map * capi.DEPTH_POINT_DTYPE.itemsize
    wall = float(np.frombuffer(raw, np.float64, 1, off)[0]); off += 8
    return fr, m, int(stopped), wall, np.frombuffer(raw, np.float64, 8, off).copy(), np.frombuffer(raw, np.uint64, 8, off + 64).copy()


def write_script(path, W, H, node_kw, ops):
    """ops: ("L" | "R", events dict), ("TS", stamp), ("POSE", stamp, T), ("PASS",)."""
    import struct
    k = node_kw
    with open(path, "wb") as f:
        f.write(struct.pack("<8id", W, H, k["mode"], k["pen"], k["ts_len"], k["em_num"], int(k["denoising"]), int(k["marker"]), k["half"]))
        f.write(struct.pack("<i", len(ops)))
        for op in ops:
            if op[0] in ("L", "R"):
                e = op[1]
                f.write(struct.pack("<ii", 0 if op[0] == "L" else 1, e["x"].size))
                for a, dt in ((e["x"], np.uint16), (e["y"], np.uint16), (e["t"], np.int64), (e["p"], np.uint8)):
                    f.write(np.ascontiguousarray(a, dt).tobytes())
            elif op[0] == "TS":
                f.write(struct.pack("<iq", 2, op[1]))
            elif op[0] == "POSE":
                f.write(struct.pack("<iq", 3, op[1])); f.write(np.ascontiguousarray(op[2], np.float64).tobytes())
            else:
                f.write(struct.pack("<i", 4))


EV_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("t", "<i8")])


def parse_dump(path, n_ops):
    """examples/mvstereo_node_dump.cpp's output -> list of dicts, one per op."""
    raw = open(path, "rb").read()
    off, out = 0, []
    for _ in range(n_ops):
        kind, reset = np.frombuffer(raw, np.int32, 2, off); off += 8
        d = dict(kind=int(kind), reset=bool(reset))
        if kind == 4:
            g, tr, h = np.frombuffer(raw, np.int32, 3, off); off += 12
            d.update(gated=bool(g), transferred=bool(tr), has_obs=bool(h))
            d["t_obs"] = int(np.frombuffer(raw, np.int64, 1, off)[0]); off += 8
            d["T_obs"] = np.frombuffer(raw, np.float64, 16, off).copy(); off += 128
            d["t_low"], d["t_up"] = [int(v) for v in np.frombuffer(raw, np.int64, 2, off)]; off += 16
            for name in ("em_left", "em_right", "sgm", "window", "close"):
                n = int(np.frombuffer(raw, np.int32, 1, off)[0]); off += 4
                d[name] = np.frombuffer(raw, EV_DTYPE, n, off).copy(); off += n * EV_DTYPE.itemsize
            n = int(np.frombuffer(raw, np.int32, 1, off)[0]); off += 4
            st = np.frombuffer(raw, np.dtype([("t", "<i8"), ("T", "<f8", (16,))]), n, off).copy(); off += n * 136
            d["st_t"], d["st_T"] = st["t"], st["T"]
        out.append(d)
    assert off == len(raw)
    return out


def run_script(W, H, node_kw, ops):
    """The same script through Node: a list of dicts shaped like parse_dump's."""
    n = Node(W, H, node_kw["mode"], node_kw["pen"], node_kw["ts_len"], node_kw["em_num"], node_kw["half"], node_kw["denoising"], node_kw["marker"])
    zeros = np.zeros((H, W), np.uint8)
    out = []
    ev = lambda e: np.array(list(zip(e["x"], e["y"], e["t"])), EV_DTYPE)
    for op in ops:
        if op[0] in ("L", "R"):
            out.append(dict(kind=0 if op[0] == "L" else 1, reset=n.events(op[1], op[0] == "L")))
        elif op[0] == "TS":
            out.append(dict(kind=2, reset=n.time_surface(op[1], zeros, zeros)))
        elif op[0] == "POSE":
            out.append(dict(kind=3, reset=n.pose(op[1], op[2])))
        else:
            g, tr, h = n.prepare()
            d = dict(kind=4, reset=False, gated=g, transferred=tr, has_obs=h)
            d["t_obs"] = n.obs[0] if n.obs else 0
            d["T_obs"] = n.obs[1].ravel() if n.obs else np.zeros(16)
            d["t_low"], d["t_up"] = n.t_low, n.t_up
            for name in ("em_left", "em_right", "sgm", "window", "close"):
                d[name] = ev(getattr(n, name))
            d["st_t"], d["st_T"] = n.st_t, n.st_T
            # coverage marks (restatement only): the SGM walk started one past the newest event; a pose sample was skipped
            lb = n.left.lower_bound(d["t_obs"])
            t_begin = ind.ros_from_sec(max(0.0, ind.ros_to_sec(d["t_obs"]) - 2 * n.half))
            d["sgm_past_end"] = bool(h and n.mode == 4 and lb == n.left.t.size and n.left.lower_bound(t_begin) < lb)
            d["pose_miss"] = bool(h and n.mode in (1, 3) and n.st_t.size < ind.sample_pose_stamps(d["t_obs"], n.half).size)
            d["em_right_window"] = n.right.lower_bound(n.t_up) - n.right.lower_bound(n.t_low) if h and n.mode in (0, 2) else -1
            out.append(d)
    return out
