"""Independent restatement of the closed ESVO loop (include/esvo_b200/esvo_system.hpp), written from the REFERENCE sources:
esvo_core/src/esvo_Mapping.cpp (MappingLoop :179-259, dataTransferring :494-605, callbacks :607-762, publishMappingResults /
publishPointCloud :868-953), esvo_core/src/esvo_Tracking.cpp (TrackingLoop :79-200, refDataTransferring / curDataTransferring
:202-265, callbacks :279-373, saveTrajectory :430-462) and the tf2 TimeCache behaviour both nodes rely on (DESIGN.md section 2).
Drives any capi.Backend: the per-pixel stages run through the C ABI, everything node-level is plain Python here.  The SGM of
InitializationAtTime is a callable (the Backend's sgbm_compute on the product, cv2.StereoSGBM on the oracle).
TEST INFRASTRUCTURE: clarity over speed.
"""
import ctypes as C
import math

import numpy as np

import indep_numpy as ind

IDENTITY = np.eye(4)
STATUS_CODE = {"INITIALIZATION": 0, "WORKING": 1, "TERMINATE": 2}
# the loop's tick record and mapping record (layout of examples/system_loop.cpp's result file)
TICK_DTYPE = np.dtype([("t", "<i8"), ("status", "<i4"), ("has_pose", "<i4"), ("T", "<f8", (16,)), ("ms", "<f8", (3,))])
MAP_DTYPE = np.dtype([("tick", "<i4"), ("ran", "<i4"), ("ok", "<i4"), ("published", "<i4"), ("n_sgm_points", "<u8"),
                      ("ctr", "<u8", (8,)), ("cloud_points", "<u8"), ("stamp", "<i8")])
CTR_KEYS = ("n_events", "n_seeds", "n_solved", "n_culled", "n_fusions", "bm_evals", "lm_evals", "map_size")


# ---- the pose hand-off: Eigen::Quaterniond(Matrix3d) / toRotationMatrix (Eigen/src/Geometry/Quaternion.h) ----
def quat_from_rot(m):
    """quaternion_assign_impl: returns (x, y, z, w)."""
    m = np.asarray(m, float)
    q = [0.0, 0.0, 0.0, 0.0]
    t = float(m[0, 0]) + float(m[1, 1]) + float(m[2, 2])
    if t > 0:
        t = math.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0] = (m[2, 1] - m[1, 2]) * t; q[1] = (m[0, 2] - m[2, 0]) * t; q[2] = (m[1, 0] - m[0, 1]) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j = (i + 1) % 3; k = (j + 1) % 3
        t = math.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (m[k, j] - m[j, k]) * t; q[j] = (m[j, i] + m[i, j]) * t; q[k] = (m[k, i] + m[i, k]) * t
    return [float(v) for v in q]


def rot_from_quat(q):
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def slerp_tf2(a, b, t):
    """tf2::Quaternion::slerp with angleShortestPath; tf2Acos clamps its argument to [-1, 1]."""
    dot = lambda u, v: u[0] * v[0] + u[1] * v[1] + u[2] * v[2] + u[3] * v[3]
    s = math.sqrt(dot(a, a) * dot(b, b)); d_ab = dot(a, b)
    theta = math.acos(max(-1.0, min(1.0, abs(d_ab) / s))) * 2.0 / 2.0
    if theta == 0.0:
        return list(a)
    d = 1.0 / math.sin(theta); s0 = math.sin((1.0 - t) * theta); s1 = math.sin(t * theta)
    sg = -1.0 if d_ab < 0 else 1.0
    return [(a[i] * s0 + sg * b[i] * s1) * d for i in range(4)]


class PoseBuffer:
    """tf::Transformer(true, ros::Duration(100.0)) as the nodes use it: stampedPoseCallback -> setTransform, getPoseAt ->
    canTransform + lookupTransform + transformTFToKindr."""

    def __init__(self, cache_ns=100 * 10**9):
        self.cache = cache_ns
        self.t, self.q, self.p = [], [], []        # oldest first

    def set_transform(self, t_ns, T):
        t_ns = int(t_ns)
        if self.t and self.t[-1] > t_ns + self.cache:
            return False
        i = int(np.searchsorted(np.array(self.t, np.int64), t_ns, side="left")) if self.t else 0
        if i < len(self.t) and self.t[i] == t_ns:
            return False
        T = np.asarray(T, float).reshape(4, 4)
        self.t.insert(i, t_ns); self.q.insert(i, quat_from_rot(T[:3, :3])); self.p.insert(i, [float(v) for v in T[:3, 3]])
        while self.t[0] + self.cache < self.t[-1]:
            del self.t[0], self.q[0], self.p[0]
        return True

    def lookup(self, t_ns):
        """T_world_dvs (4x4) at t_ns, or None where tf's canTransform is false."""
        t_ns = int(t_ns)
        if not self.t:
            return None
        if t_ns == 0:
            return self._pose(self.q[-1], self.p[-1])
        if t_ns < self.t[0] or t_ns > self.t[-1]:
            return None
        i = int(np.searchsorted(np.array(self.t, np.int64), t_ns, side="right")) - 1
        if self.t[i] == t_ns:
            return self._pose(self.q[i], self.p[i])
        r = ind.ros_to_sec(t_ns - self.t[i]) / ind.ros_to_sec(self.t[i + 1] - self.t[i])
        p = [(1.0 - r) * self.p[i][k] + r * self.p[i + 1][k] for k in range(3)]
        return self._pose(slerp_tf2(self.q[i], self.q[i + 1], r), p)

    @staticmethod
    def _pose(q, p):
        T = np.eye(4)
        T[:3, :3] = rot_from_quat(q); T[:3, 3] = p
        return T


def pack_cloud(p_cam, T):
    """publishPointCloud (:925-929): R p_cam + t per element, summed left to right like the C++ shim (frontend::packPointCloud),
    so that both give the same f32 cloud bit for bit (ind.pack_point_cloud's matrix product may sum in another order)."""
    p = np.asarray(p_cam, float).reshape(-1, 3); T = np.asarray(T, float).reshape(4, 4)
    rows = [T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1] + T[r, 2] * p[:, 2] + T[r, 3] for r in range(3)]
    return np.stack(rows, axis=1).astype(np.float32)


def fusion_window(be):
    """(dqvDepthPoints_.size(), points in it), read from the context with esvo_window_download probes."""
    k, total = 0, 0
    while True:
        n = C.c_size_t(0)
        rc = be._call("window_download", [C.c_int, C.c_void_p, C.POINTER(C.c_size_t)], k, None, C.byref(n), ok=(0, -1, -4))
        if rc not in (0, -4):
            return k, total
        total += n.value; k += 1


class Mapper:
    """esvo_Mapping without ROS."""

    def __init__(self, be, sgbm, pen, half_slice, ts_history_len, init_threshold, denoising):
        self.be, self.sgbm = be, sgbm
        self.pen, self.half, self.hist_len, self.init_thr, self.denoising = pen, half_slice, ts_history_len, init_threshold, denoising
        self.ts = {}                       # TS_history_: stamp -> (left, right)
        self.left = None                   # events_left_: (x, y, t) arrays of the delivered prefix

    def time_surface(self, t, tl, tr):
        self.ts[t] = (tl, tr)
        while len(self.ts) > self.hist_len:
            del self.ts[min(self.ts)]

    def _window(self, t_end, span_s):
        """The delivered left events from ~1 ms before t_end - span on: every selection below looks only at lower bounds
        inside that range, so the indices relative to this suffix are those of the whole buffer."""
        x, y, t = self.left
        lo = max(0, int(np.searchsorted(t, t_end - int(span_s * 1e9) - 1_000_000, side="left")) - 1)
        return x[lo:], y[lo:], t[lo:]

    def data_transferring(self, status, poses):
        """:494-605.  Returns (stamp, left, right, T_obs, events (x, y, t), st stamps, st poses) or None."""
        if len(self.ts) <= 10:
            return None
        stamps = sorted(self.ts)
        obs = None
        i = len(stamps) - 2                                       # the second-newest entry (:502-503)
        while obs is None:
            if status == "INITIALIZATION":
                obs = (stamps[i], IDENTITY.copy())
            if status == "WORKING":
                T = poses.lookup(stamps[i])
                if T is not None:
                    obs = (stamps[i], T)
            if i == 0:
                break
            i -= 1
        if obs is None:
            return None
        t_obs, T_obs = obs
        tl, tr = self.ts[t_obs]
        if status == "INITIALIZATION":                            # :537-552
            x, y, t = self._window(t_obs, 2 * self.half)
            sel = ind.select_sgm_events(t, t_obs, self.half, self.pen)
            return t_obs, tl, tr, T_obs, (x[sel], y[sel], t[sel]), None, None
        x, y, t = self._window(t_obs, 10 * self.half)              # :554-603
        sel = ind.select_close_events(t, t_obs, self.half, self.pen)
        st, sp = [], []
        for s in ind.sample_pose_stamps(t_obs, self.half):
            T = poses.lookup(s)
            if T is not None:
                st.append(s); sp.append(T.ravel())
        return t_obs, tl, tr, T_obs, (x[sel], y[sel], t[sel]), np.array(st, np.int64), np.array(sp).reshape(-1, 16)

    def denoise(self, ev):
        """createDenoisingMask / extractDenoisedEvents (:1046-1072): event map of vALLEventsPtr_left_ (= the close events),
        cv::medianBlur 3x3, keep the close events on surviving pixels, at most PROCESS_EVENT_NUM."""
        import cv2
        x, y, t = ev
        img = np.zeros((self.be.H, self.be.W), np.uint8)
        img[y.astype(int), x.astype(int)] = 255
        mask = cv2.medianBlur(img, 3)
        keep = np.nonzero(mask[y.astype(int), x.astype(int)] == 255)[0][: self.pen]
        return x[keep], y[keep], t[keep]

    def loop_once(self, status, poses):
        """One pass of MappingLoop (:194-248).  Returns a MAP_DTYPE-shaped dict and the published (stamp, cloud) or None."""
        rec = dict(ran=0, ok=0, published=0, n_sgm_points=0, ctr=[0] * 8, cloud_points=0, stamp=0)
        if status == "TERMINATE" or len(self.ts) < 10:
            return rec, None
        d = self.data_transferring(status, poses)
        if d is None:
            return rec, None
        t_obs, tl, tr, T_obs, ev, st, sp = d
        be = self.be
        if status == "INITIALIZATION":                            # InitializationAtTime (:433-492)
            rec["ran"] = 1
            disp = self.sgbm(tl, tr)
            n, acc = be.init_from_disparity(disp, ev[0], ev[1], T_obs, self.init_thr)
            rec["n_sgm_points"], rec["ok"] = n, int(acc)
        if status == "WORKING":                                   # MappingAtTime (:261-431)
            rec["ran"] = 2
            if self.denoising:
                ev = self.denoise(ev)
            else:
                ev = tuple(a[: self.pen] for a in ev)
            be.set_ts_pair(tl, tr, T_obs)
            c = be.mapping_at_time(ev[0], ev[1], ev[2], st, sp)
            rec["ctr"] = [c[k] for k in CTR_KEYS]; rec["ok"] = 1
        if not rec["ok"]:
            return rec, None
        publish = status == "INITIALIZATION"                      # publishMappingResults (:889-906)
        if status == "WORKING":
            n_frames, n_points = fusion_window(be)
            p = be.params
            publish = n_frames == p.max_num_fusion_frames if p.fusion_strategy == 0 else n_points > 0.5 * p.max_num_fusion_points
        if not publish:
            return rec, None
        cloud = pack_cloud(be.map_download()["p_cam"], T_obs)
        if cloud.shape[0] == 0:                                   # :945
            return rec, None
        rec["published"], rec["cloud_points"], rec["stamp"] = 1, cloud.shape[0], t_obs
        return rec, (t_obs, cloud)


class Tracker:
    """esvo_Tracking without ROS (RegProblemType analytical, tracking_hkust.yaml)."""

    def __init__(self, be, ts_history_len=100, ref_history_len=10):
        self.be, self.ts_len, self.ref_len = be, ts_history_len, ref_history_len
        self.ets = "IDLE"
        self.ref_maps = {}                 # refPCMap_
        self.ts = {}                       # TS_history_ (left images)
        self.ref_t, self.ref_T, self.ref_xyz = 0, IDENTITY.copy(), None
        self.cur_t, self.cur_T = 0, IDENTITY.copy()
        self.T_world_cur = IDENTITY.copy()
        self.traj = []                     # (stamp, T) of every tracked frame (lTimestamp_ / lPose_)

    def ref_map(self, t, cloud):
        self.ref_maps[t] = cloud
        while len(self.ref_maps) > self.ref_len:
            del self.ref_maps[min(self.ref_maps)]

    def time_surface(self, t, tl):
        self.ts[t] = tl
        while len(self.ts) > self.ts_len:
            del self.ts[min(self.ts)]

    def loop_once(self, status, poses):
        """One pass of TrackingLoop (:84-184).  Returns (status, pose or None, error or None)."""
        sec = ind.ros_to_sec
        if len(self.ref_maps) < 1 or len(self.ts) < 1:
            return status, None, None
        if status == "INITIALIZATION" and self.ets == "WORKING":  # :92-97
            self.ets = "IDLE"; self.ts.clear(); self.ref_maps.clear()
            return status, None, None
        if status == "TERMINATE":
            return status, None, None
        t_ref_new, t_ts_new = max(self.ref_maps), max(self.ts)
        if sec(self.ref_t) < sec(t_ref_new):                       # refDataTransferring (:202-234)
            self.ref_t = t_ref_new
            if status == "INITIALIZATION" and self.ets == "IDLE":
                self.ref_T = IDENTITY.copy()
            if status == "WORKING" or (status == "INITIALIZATION" and self.ets == "WORKING"):
                T = poses.lookup(self.ref_t)
                if T is None:
                    return status, None, "no pose for the reference map"
                self.ref_T = T
            self.ref_xyz = np.ascontiguousarray(self.ref_maps[t_ref_new], np.float32).copy()
        if sec(self.cur_t) < sec(t_ts_new):
            if sec(self.ref_t) >= sec(t_ts_new):
                return status, None, "time-surface observation is not newer than the reference map"
            if self.cur_t == t_ts_new:                             # curDataTransferring (:236-265)
                return status, None, None
            self.cur_t = t_ts_new
            if status == "INITIALIZATION" and self.ets == "IDLE":
                self.cur_T = self.ref_T.copy()
            if status == "WORKING" or (status == "INITIALIZATION" and self.ets == "WORKING"):
                self.cur_T = self.T_world_cur.copy()
        else:
            return status, None, None
        if self.be.track_reset(self.ref_xyz, self.ref_T, self.cur_T, self.ts[self.cur_t]) == 0:
            self.ets = "WORKING"
            status = "WORKING"
            try:                                                  # fails only on a device / ABI error: the system stops
                T, _ = self.be.track_solve(True)
            except Exception as e:                                # capi.EsvoError
                return status, None, f"tracking solve: {e}"
            self.cur_T = T.copy(); self.T_world_cur = T.copy()
            self.traj.append((self.cur_t, T.copy()))
            return status, T.copy(), None
        self.ets = "IDLE"
        return "INITIALIZATION", None, None


def run_system(be, sgbm, left, right, t0_ns, dt_ns, n_ticks, mapping_every=5, pen=1000, half_slice=0.001, init_threshold=500,
               denoising=True, ts_history_len=100, trk_ts_history_len=100, ref_history_len=10):
    """The fixed schedule of esvo_core::esvo_System (DESIGN.md section 5) on one Backend.  left / right: dicts of x, y, t, p
    (time-ordered).  Returns (ticks: TICK_DTYPE array, mapping: MAP_DTYPE array, final map, trajectory, error)."""
    be.track_srand(1)
    mapper = Mapper(be, sgbm, pen, half_slice, ts_history_len, init_threshold, denoising)
    tracker = Tracker(be, trk_ts_history_len, ref_history_len)
    poses = PoseBuffer()
    status, error = "INITIALIZATION", None
    ticks, maps = [], []
    done = [0, 0]
    for k in range(n_ticks):
        t = t0_ns + k * dt_ns
        for cam, e in enumerate((left, right)):                   # 1. events with stamp < t_k
            hi = int(np.searchsorted(e["t"], t, side="left"))
            if hi > done[cam]:
                sl = slice(done[cam], hi)
                be.ts_push_events(cam, e["x"][sl], e["y"][sl], e["t"][sl], e["p"][sl])
            done[cam] = hi
        mapper.left = (left["x"][: done[0]], left["y"][: done[0]], left["t"][: done[0]])
        _, tl = be.ts_build(0, t, want_idx=False)                  # 2. both time surfaces at t_k
        _, tr = be.ts_build(1, t, want_idx=False)
        mapper.time_surface(t, tl, tr); tracker.time_surface(t, tl)
        rec = np.zeros((), TICK_DTYPE); rec["t"] = t
        status, T, error = tracker.loop_once(status, poses)       # 3. tracking; the pose goes to tf at once
        if error is not None:
            status = "TERMINATE"
        elif T is not None:
            rec["has_pose"] = 1; rec["T"] = T.ravel()
            poses.set_transform(t, T)
        if error is None and k % mapping_every == 0:              # 4. mapping; the map goes to refMapCallback
            m, pub = mapper.loop_once(status, poses)
            mr = np.zeros((), MAP_DTYPE); mr["tick"] = k
            for key, v in m.items():
                mr[key] = v
            maps.append(mr)
            if pub is not None:
                tracker.ref_map(*pub)
        rec["status"] = STATUS_CODE[status]
        ticks.append(rec)
        if error is not None:
            break
    return np.array(ticks, TICK_DTYPE), np.array(maps, MAP_DTYPE), be.map_download(), tracker.traj, error


def parse_result(path):
    """examples/system_loop.cpp's result file -> (ticks, mapping, map, stopped, wall_ms, stage_ms, stage_launches)."""
    from esvo_b200 import capi
    raw = open(path, "rb").read()
    n_t, n_m, n_map, stopped = np.frombuffer(raw, np.int32, 4)
    off = 16
    ticks = np.frombuffer(raw, TICK_DTYPE, n_t, off).copy(); off += n_t * TICK_DTYPE.itemsize
    maps = np.frombuffer(raw, MAP_DTYPE, n_m, off).copy(); off += n_m * MAP_DTYPE.itemsize
    m = np.frombuffer(raw, capi.DEPTH_POINT_DTYPE, n_map, off).copy(); off += n_map * capi.DEPTH_POINT_DTYPE.itemsize
    wall = float(np.frombuffer(raw, np.float64, 1, off)[0]); off += 8
    prof_ms = np.frombuffer(raw, np.float64, 8, off).copy(); off += 64
    prof_n = np.frombuffer(raw, np.uint64, 8, off).copy()
    return ticks, maps, m, int(stopped), wall, prof_ms, prof_n


def write_scenario(path, W, H, t0_ns, dt_ns, n_ticks, left, right, mapping_every=5, profile=False, overrides=()):
    """The scenario examples/system_loop.cpp reads.  overrides: (key, value) with keys 0 trk_batch_size, 1 PROCESS_EVENT_NUM,
    2 Denoising, 3 INIT_SGM_DP_NUM_THRESHOLD."""
    import struct
    with open(path, "wb") as f:
        f.write(struct.pack("<iii", W, H, 0)); f.write(struct.pack("<qq", t0_ns, dt_ns))
        f.write(struct.pack("<iiii", n_ticks, mapping_every, int(profile), len(overrides)))
        for key, v in overrides:
            f.write(struct.pack("<id", key, float(v)))
        for e in (left, right):
            f.write(struct.pack("<i", e["x"].size))
            for a, dt in ((e["x"], np.uint16), (e["y"], np.uint16), (e["t"], np.int64), (e["p"], np.uint8)):
                f.write(np.ascontiguousarray(a, dt).tobytes())


def read_trajectory(path):
    """saveTrajectory's text file -> (stamp seconds, 7-vectors tx ty tz qx qy qz qw)."""
    rows = [ln.split() for ln in open(path) if ln.strip()]
    return np.array([float(r[0]) for r in rows]), np.array([[float(v) for v in r[1:]] for r in rows]).reshape(-1, 7)


def trajectory_errors(ticks, gt_at, t_align_ns):
    """ATE (RMS of the position error) and the largest rotation error (degrees) of the tracked poses against ground truth
    gt_at(t_ns) -> T_world_left, aligned at t_align_ns (the SGM start-up frame, where the system's world is the left camera)."""
    G0inv = np.linalg.inv(gt_at(t_align_ns))
    pos, rot = [], []
    for r in ticks[ticks["has_pose"] == 1]:
        G = G0inv @ gt_at(int(r["t"])); T = r["T"].reshape(4, 4)
        pos.append(np.linalg.norm(T[:3, 3] - G[:3, 3]))
        c = (np.trace(G[:3, :3].T @ T[:3, :3]) - 1) / 2
        rot.append(np.degrees(np.arccos(np.clip(c, -1, 1))))
    if not pos:
        return float("inf"), float("inf")
    return float(np.sqrt(np.mean(np.square(pos)))), float(np.max(rot))
