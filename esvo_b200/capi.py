"""ctypes binding of the C ABI declared in include/esvo_b200.h.

The `Backend` class binds any library that exports the ABI under some prefix:
  * the product library  esvo_b200/_build/libesvo_b200.so   (prefix "esvo_",  CUDA, sm_90a) -- load_product() below;
  * the CPU oracle (prefix "esvo_oracle_") is loaded by oracle/loader.py, which lives OUTSIDE this package (test infrastructure).

The product path never falls back to the oracle: `load_product()` raises if the CUDA library
is missing, and `esvo_create` fails with ESVO_ERR_NO_DEVICE when there is no usable GPU.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT_LIB = os.path.join(_ROOT, "esvo_b200", "_build", "libesvo_b200.so")

ESVO_OK = 0
ERR_NAMES = {0: "OK", -1: "INVALID_ARG", -2: "NO_DEVICE", -3: "CUDA", -4: "CAPACITY", -5: "STATE",
             -6: "UNSUPPORTED"}
DIST_PLUMB_BOB, DIST_EQUIDISTANT = 0, 1
LSNORM_L2, LSNORM_TDIST, LSNORM_ZNCC = 0, 1, 2
TRK_L2, TRK_HUBER = 0, 1
FUSION_CONST_FRAMES, FUSION_CONST_POINTS = 0, 1


class Calib(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("distortion_model", C.c_int32),
                ("_pad", C.c_int32), ("K", C.c_double * 9), ("D", C.c_double * 4),
                ("R", C.c_double * 9), ("P", C.c_double * 12)]


class Params(C.Structure):
    _fields_ = [
        ("decay_ms", C.c_double), ("ignore_polarity", C.c_int32),
        ("median_blur_kernel_size", C.c_int32), ("max_event_queue_len", C.c_int32),
        ("time_surface_mode", C.c_int32),
        ("patch_size_x", C.c_int32), ("patch_size_y", C.c_int32),
        ("bm_min_disparity", C.c_int32), ("bm_max_disparity", C.c_int32),
        ("bm_step", C.c_int32), ("bm_updown", C.c_int32), ("smooth_time_surface", C.c_int32),
        ("bm_zncc_threshold", C.c_double),
        ("lsnorm", C.c_int32), ("max_iteration", C.c_int32),
        ("td_nu", C.c_double), ("td_scale", C.c_double),
        ("invdepth_min_range", C.c_double), ("invdepth_max_range", C.c_double),
        ("residual_vis_threshold", C.c_double), ("stdvar_vis_threshold", C.c_double),
        ("age_vis_threshold", C.c_double),
        ("fusion_radius", C.c_int32), ("fusion_strategy", C.c_int32),
        ("max_num_fusion_frames", C.c_int32), ("max_num_fusion_points", C.c_int32),
        ("regularization", C.c_int32), ("reg_radius", C.c_int32),
        ("reg_min_neighbours", C.c_int32), ("reg_min_close_neighbours", C.c_int32),
        ("trk_patch_size_x", C.c_int32), ("trk_patch_size_y", C.c_int32),
        ("trk_kernel_size", C.c_int32), ("trk_lsnorm", C.c_int32),
        ("trk_huber_threshold", C.c_double),
        ("trk_max_registration_points", C.c_int32), ("trk_batch_size", C.c_int32),
        ("trk_max_iteration", C.c_int32), ("trk_min_num_events", C.c_int32),
        ("num_thread_mapping", C.c_int32), ("_pad", C.c_int32),
    ]


class EmParams(C.Structure):
    """esvo_em_params (include/esvo_b200.h): EventMatcher thresholds / patch size / thread count."""
    _fields_ = [("time_threshold_s", C.c_double), ("epipolar_threshold", C.c_double), ("ts_ncc_threshold", C.c_double),
                ("patch_size_x", C.c_int32), ("patch_size_y", C.c_int32), ("num_thread", C.c_int32), ("_pad", C.c_int32)]


class LMStats(C.Structure):
    _fields_ = [("n_points", C.c_int64), ("nfev", C.c_int64), ("n_iter", C.c_int64)]


# numpy mirrors of the POD structs (C layout, no padding surprises: all 8-byte aligned)
SEED_DTYPE = np.dtype([
    ("x_left_raw", "<f8", (2,)), ("x_left", "<f8", (2,)), ("x_right", "<f8", (2,)),
    ("t_ns", "<i8"), ("T_world_virtual", "<f8", (16,)),
    ("inv_depth", "<f8"), ("cost", "<f8"), ("disp", "<f8")], align=True)
DEPTH_POINT_DTYPE = np.dtype([
    ("row", "<i4"), ("col", "<i4"), ("x", "<f8", (2,)), ("inv_depth", "<f8"), ("scale2", "<f8"),
    ("nu", "<f8"), ("variance", "<f8"), ("residual", "<f8"), ("age", "<i8"),
    ("p_cam", "<f8", (3,)), ("T_world_cam", "<f8", (16,))], align=True)
assert SEED_DTYPE.itemsize == 8 * (2 + 2 + 2 + 1 + 16 + 3)
assert DEPTH_POINT_DTYPE.itemsize == 8 + 8 * (2 + 5 + 1 + 3 + 16)
# dvs_msgs/Event as serialised in a ROS bag (esvo_ts_push_event_array): packed, little-endian, 13 bytes
EVENT_WIRE_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("sec", "<u4"), ("nsec", "<u4"), ("polarity", "u1")])
assert EVENT_WIRE_DTYPE.itemsize == 13

# The 8-counter record of a mapping frame, in the order the C ABI writes it (esvo_fetch_mapping_counters, esvo_results_end)
MAPPING_COUNTER_KEYS = ("n_events", "n_seeds", "n_solved", "n_culled", "n_fusions", "bm_evals", "lm_evals", "map_size")


def _mapping_counters(ctr) -> dict:
    return dict(zip(MAPPING_COUNTER_KEYS, [int(v) for v in ctr]))


def pack_events(x, y, t_ns, pol):
    """SoA events -> wire records (stamp split as ros::Time: sec = t // 1e9, nsec = t % 1e9); pol bytes are kept as given."""
    t = np.asarray(t_ns, np.int64)
    r = np.empty(t.size, EVENT_WIRE_DTYPE)
    r["x"] = x; r["y"] = y; r["sec"] = t // 1_000_000_000; r["nsec"] = t % 1_000_000_000; r["polarity"] = pol
    return r


class EsvoError(RuntimeError):
    def __init__(self, code, where, msg=""):
        super().__init__(f"{where}: {ERR_NAMES.get(code, code)} {msg}")
        self.code = code


def _ptr(a, ctype):
    if a is None:
        return None
    return a.ctypes.data_as(C.POINTER(ctype))


def _arr(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def _wire_runs(runs):
    """Byte buffers of whole wire records -> (the buffers as uint8 arrays, void* array, size_t record counts)."""
    bufs = [np.frombuffer(r, np.uint8) if not isinstance(r, np.ndarray) else _arr(r, np.uint8).ravel() for r in runs]
    for b in bufs:
        assert b.size % EVENT_WIRE_DTYPE.itemsize == 0
    ptrs = (C.c_void_p * max(1, len(bufs)))(*[b.ctypes.data if b.size else None for b in bufs])
    ns = (C.c_size_t * max(1, len(bufs)))(*[b.size // EVENT_WIRE_DTYPE.itemsize for b in bufs])
    return bufs, ptrs, ns


@dataclass
class Library:
    lib: C.CDLL
    prefix: str
    path: str

    def fn(self, name):
        return getattr(self.lib, self.prefix + name)


def load_product() -> Library:
    if not os.path.exists(PRODUCT_LIB):
        raise RuntimeError(
            f"{PRODUCT_LIB} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the product path)")
    return Library(C.CDLL(PRODUCT_LIB), "esvo_", PRODUCT_LIB)


def default_params(lib: Library) -> Params:
    p = Params()
    f = lib.fn("default_params")
    f.argtypes = [C.POINTER(Params)]
    f.restype = None
    f(C.byref(p))
    return p


def compute_rectify_tables(lib: Library, calib: Calib):
    """esvo_compute_rectify_tables: the product's own host-side tables for one camera (no context, no GPU)."""
    n = calib.width * calib.height
    m1 = np.empty(n, np.float32); m2 = np.empty(n, np.float32); lut = np.empty(2 * n, np.float64); mask = np.empty(n, np.uint8)
    f = lib.fn("compute_rectify_tables")
    f.argtypes = [C.POINTER(Calib), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_uint8)]
    f.restype = C.c_int
    rc = f(C.byref(calib), _ptr(m1, C.c_float), _ptr(m2, C.c_float), _ptr(lut, C.c_double), _ptr(mask, C.c_uint8))
    if rc:
        raise EsvoError(rc, "compute_rectify_tables")
    H, W = calib.height, calib.width
    return m1.reshape(H, W), m2.reshape(H, W), lut.reshape(H, W, 2), mask.reshape(H, W)


def make_calib(width, height, model, K, D, R, P) -> Calib:
    c = Calib()
    c.width, c.height = int(width), int(height)
    c.distortion_model = DIST_EQUIDISTANT if model in (1, "equidistant") else DIST_PLUMB_BOB
    for dst, src, n in ((c.K, K, 9), (c.D, D, 4), (c.R, R, 9), (c.P, P, 12)):
        src = np.asarray(src, dtype=np.float64).ravel()
        assert src.size == n
        for i in range(n):
            dst[i] = float(src[i])
    return c


class Backend:
    """One esvo_ctx (or esvo_oracle_ctx).  Method names follow the C ABI."""

    def __init__(self, lib: Library, left: Calib, right: Calib, params: Params, device: int = 0):
        self.L = lib
        self.W, self.H = left.width, left.height
        self.params = params
        st = C.c_int(0)
        f = lib.fn("create")
        f.argtypes = [C.c_int, C.POINTER(Calib), C.POINTER(Calib), C.POINTER(Params), C.POINTER(C.c_int)]
        f.restype = C.c_void_p
        self.ctx = f(device, C.byref(left), C.byref(right), C.byref(params), C.byref(st))
        if not self.ctx:
            raise EsvoError(st.value, "create")
        self.ctx = C.c_void_p(self.ctx)

    def _call(self, name, argtypes, *args, ok=(0,)):
        cache = self.__dict__.setdefault("_fn_cache", {})
        f = cache.get(name)
        if f is None:                      # prototypes are set once per entry point (this sits on the per-frame path)
            f = self.L.fn(name)
            f.argtypes = [C.c_void_p] + list(argtypes)
            f.restype = C.c_int
            cache[name] = f
        rc = f(self.ctx, *args)
        if rc not in ok:
            msg = ""
            if self.L.prefix == "esvo_":
                g = self.L.fn("last_error")
                g.argtypes = [C.c_void_p]
                g.restype = C.c_char_p
                msg = (g(self.ctx) or b"").decode()
            raise EsvoError(rc, name, msg)
        return rc

    def close(self):
        if self.ctx:
            f = self.L.fn("destroy")
            f.argtypes = [C.c_void_p]
            f.restype = None
            f(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- tables ----
    def set_rectify_tables(self, cam, map1=None, map2=None, lut=None, mask=None):
        m1 = None if map1 is None else _arr(map1, np.float32)
        m2 = None if map2 is None else _arr(map2, np.float32)
        lu = None if lut is None else _arr(lut, np.float64)
        mk = None if mask is None else _arr(mask, np.uint8)
        self._call("set_rectify_tables",
                   [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_uint8)],
                   cam, _ptr(m1, C.c_float), _ptr(m2, C.c_float), _ptr(lu, C.c_double), _ptr(mk, C.c_uint8))

    def get_rectify_tables(self, cam):
        n = self.W * self.H
        m1 = np.empty(n, np.float32); m2 = np.empty(n, np.float32)
        lut = np.empty(2 * n, np.float64); mask = np.empty(n, np.uint8)
        self._call("get_rectify_tables",
                   [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_uint8)],
                   cam, _ptr(m1, C.c_float), _ptr(m2, C.c_float), _ptr(lut, C.c_double), _ptr(mask, C.c_uint8))
        return (m1.reshape(self.H, self.W), m2.reshape(self.H, self.W), lut.reshape(self.H, self.W, 2),
                mask.reshape(self.H, self.W))

    def get_derived(self):
        out = (C.c_double * 4)()
        self._call("get_derived", [C.POINTER(C.c_double)], out)
        return dict(baseline=out[0], min_disparity=int(out[1]), max_disparity=int(out[2]), td_stdvar=out[3])

    # ---- time surface ----
    def ts_push_events(self, cam, x, y, t_ns, pol):
        x = _arr(x, np.uint16); y = _arr(y, np.uint16); t = _arr(t_ns, np.int64); p = _arr(pol, np.uint8)
        self._call("ts_push_events",
                   [C.c_int, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.POINTER(C.c_int64), C.POINTER(C.c_uint8), C.c_size_t],
                   cam, _ptr(x, C.c_uint16), _ptr(y, C.c_uint16), _ptr(t, C.c_int64), _ptr(p, C.c_uint8), x.size)

    def ts_build(self, cam, t_sync_ns, want_idx=True, want_ts=True):
        idx = np.empty(self.W * self.H, np.int64) if want_idx else None
        ts = np.empty(self.W * self.H, np.uint8) if want_ts else None
        self._call("ts_build", [C.c_int, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_uint8)],
                   cam, int(t_sync_ns), _ptr(idx, C.c_int64), _ptr(ts, C.c_uint8))
        return (None if idx is None else idx.reshape(self.H, self.W),
                None if ts is None else ts.reshape(self.H, self.W))

    def ts_reset(self, cam):
        self._call("ts_reset", [C.c_int], cam)

    def ts_push_event_array(self, cam, runs, ok=(0,)):
        """esvo_ts_push_event_array: runs is a list of byte buffers (bytes, bytearray, uint8 arrays), each a whole number of
        13-byte dvs_msgs/Event wire records (EVENT_WIRE_DTYPE).  Returns the return code (in ok, else EsvoError)."""
        bufs, ptrs, ns = _wire_runs(runs)
        return self._call("ts_push_event_array", [C.c_int, C.c_void_p, C.c_void_p, C.c_int], cam, C.cast(ptrs, C.c_void_p),
                          C.cast(ns, C.c_void_p), len(bufs), ok=ok)

    def ts_push_event_array_dev(self, cam, packed_dev_ptr, n, ok=(0,)):
        """esvo_ts_push_event_array_dev: n wire records at the device address packed_dev_ptr (an int, any alignment)."""
        return self._call("ts_push_event_array_dev", [C.c_int, C.c_void_p, C.c_size_t], cam, C.c_void_p(packed_dev_ptr), n, ok=ok)

    def ts_events_pushed(self, cam):
        """esvo_ts_events_pushed: events in the camera's log since create / ts_reset (with a hot-pixel mask, those kept)."""
        total = C.c_int64(0)
        self._call("ts_events_pushed", [C.c_int, C.POINTER(C.c_int64)], cam, C.byref(total))
        return total.value

    # ---- hot pixels (include/esvo_b200_hotpix.h) ----
    def hotpix_count_event_array(self, cam, runs, ok=(0,)):
        """esvo_hotpix_count_event_array: runs as for ts_push_event_array."""
        bufs, ptrs, ns = _wire_runs(runs)
        return self._call("hotpix_count_event_array", [C.c_int, C.c_void_p, C.c_void_p, C.c_int], cam, C.cast(ptrs, C.c_void_p),
                          C.cast(ns, C.c_void_p), len(bufs), ok=ok)

    def hotpix_count_event_array_dev(self, cam, packed_dev_ptr, n, ok=(0,)):
        """esvo_hotpix_count_event_array_dev: n wire records at the device address packed_dev_ptr (an int, any alignment)."""
        return self._call("hotpix_count_event_array_dev", [C.c_int, C.c_void_p, C.c_size_t], cam, C.c_void_p(packed_dev_ptr), n, ok=ok)

    def hotpix_select(self, cam, k, ok=(0,)):
        """esvo_hotpix_select -> (return code, number of hot pixels)."""
        n_hot = C.c_int64(-1)
        rc = self._call("hotpix_select", [C.c_int, C.c_double, C.POINTER(C.c_int64)], cam, float(k), C.byref(n_hot), ok=ok)
        return rc, n_hot.value

    def hotpix_read(self, cam):
        """esvo_hotpix_read -> (counts H x W u32, mask H x W u8)."""
        counts = np.empty(self.W * self.H, np.uint32); mask = np.empty(self.W * self.H, np.uint8)
        self._call("hotpix_read", [C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)], cam, _ptr(counts, C.c_uint32), _ptr(mask, C.c_uint8))
        return counts.reshape(self.H, self.W), mask.reshape(self.H, self.W)

    def hotpix_clear(self, cam):
        self._call("hotpix_clear", [C.c_int], cam)

    # ---- mapping ----
    def set_ts_pair(self, ts_left, ts_right, T_world_left):
        l = None if ts_left is None else _arr(ts_left, np.uint8)
        r = None if ts_right is None else _arr(ts_right, np.uint8)
        T = _arr(T_world_left, np.float64)
        self._call("set_ts_pair", [C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.POINTER(C.c_double)],
                   _ptr(l, C.c_uint8), _ptr(r, C.c_uint8), _ptr(T, C.c_double))

    @staticmethod
    def _ev_args(ex, ey, et, pose_t, poses):
        ex = _arr(ex, np.uint16); ey = _arr(ey, np.uint16); et = _arr(et, np.int64)
        pt = _arr(pose_t, np.int64); ps = _arr(poses, np.float64).reshape(-1, 16)
        assert ps.shape[0] == pt.size
        return ex, ey, et, pt, ps

    _EV_TYPES = [C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.POINTER(C.c_int64), C.c_size_t,
                 C.POINTER(C.c_int64), C.POINTER(C.c_double), C.c_size_t]

    def bm_match(self, ex, ey, et, pose_t, poses):
        ex, ey, et, pt, ps = self._ev_args(ex, ey, et, pose_t, poses)
        out = np.zeros(max(ex.size, 1), SEED_DTYPE)
        n = C.c_size_t(out.size); ev = C.c_uint64(0)
        self._call("bm_match", self._EV_TYPES + [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)],
                   _ptr(ex, C.c_uint16), _ptr(ey, C.c_uint16), _ptr(et, C.c_int64), ex.size,
                   _ptr(pt, C.c_int64), _ptr(ps, C.c_double), pt.size,
                   out.ctypes.data_as(C.c_void_p), C.byref(n), C.byref(ev))
        return out[: n.value].copy(), ev.value

    def depth_solve(self, seeds):
        seeds = np.ascontiguousarray(seeds, dtype=SEED_DTYPE)
        out = np.zeros(max(seeds.size, 1), DEPTH_POINT_DTYPE)
        n = C.c_size_t(out.size); ev = C.c_uint64(0)
        self._call("depth_solve", [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)],
                   seeds.ctypes.data_as(C.c_void_p), seeds.size, out.ctypes.data_as(C.c_void_p), C.byref(n), C.byref(ev))
        return out[: n.value].copy(), ev.value

    def depth_cull(self, pts, std_thr, cost_thr, rho_min, rho_max):
        pts = np.ascontiguousarray(pts, dtype=DEPTH_POINT_DTYPE).copy()
        n = C.c_size_t(pts.size)
        self._call("depth_cull", [C.c_void_p, C.POINTER(C.c_size_t), C.c_double, C.c_double, C.c_double, C.c_double],
                   pts.ctypes.data_as(C.c_void_p), C.byref(n), std_thr, cost_thr, rho_min, rho_max)
        return pts[: n.value].copy()

    def fuse(self, pts, T_world_frame, fusion_radius, reset_map):
        pts = np.ascontiguousarray(pts, dtype=DEPTH_POINT_DTYPE)
        T = _arr(T_world_frame, np.float64)
        nf = C.c_int(0)
        self._call("fuse", [C.c_void_p, C.c_size_t, C.POINTER(C.c_double), C.c_int, C.c_int, C.POINTER(C.c_int)],
                   pts.ctypes.data_as(C.c_void_p), pts.size, _ptr(T, C.c_double), fusion_radius, int(reset_map), C.byref(nf))
        return nf.value

    # ---- comparison modes of esvo_MVStereo (EventMatcher.cpp, esvo_MVStereo.cpp:257-431,1072-1097) ----
    def em_match(self, left, right, slice_counts, slice_poses, time_thr=5e-4, epi_thr=1.0, ncc_thr=0.1, patch=(15, 7), num_thread=4):
        """left / right: dicts with x, y, t (ns), p arrays (right time-ordered); slices over the left events."""
        prm = EmParams(time_thr, epi_thr, ncc_thr, patch[0], patch[1], num_thread, 0)

        def ev(d):
            return (_arr(d["x"], np.uint16), _arr(d["y"], np.uint16), _arr(d["t"], np.int64), _arr(d["p"], np.uint8))
        lx, ly, lt, lp = ev(left); rx, ry, rt, rp = ev(right)
        sc = _arr(slice_counts, np.int32); sp = _arr(slice_poses, np.float64)
        out = np.zeros(max(lx.size, 1), SEED_DTYPE)
        n = C.c_size_t(out.size); evals = C.c_uint64(0)
        E = [C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.POINTER(C.c_int64), C.POINTER(C.c_uint8), C.c_size_t]
        self._call("em_match", [C.POINTER(EmParams)] + E + [C.POINTER(C.c_int32), C.POINTER(C.c_double), C.c_size_t] + E +
                   [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)],
                   C.byref(prm), _ptr(lx, C.c_uint16), _ptr(ly, C.c_uint16), _ptr(lt, C.c_int64), _ptr(lp, C.c_uint8), lx.size,
                   _ptr(sc, C.c_int32), _ptr(sp, C.c_double), sc.size,
                   _ptr(rx, C.c_uint16), _ptr(ry, C.c_uint16), _ptr(rt, C.c_int64), _ptr(rp, C.c_uint8), rx.size,
                   out.ctypes.data_as(C.c_void_p), C.byref(n), C.byref(evals))
        return out[: n.value].copy(), evals.value

    def seeds_to_points(self, seeds):
        seeds = np.ascontiguousarray(seeds, dtype=SEED_DTYPE)
        out = np.zeros(max(seeds.size, 1), DEPTH_POINT_DTYPE)
        self._call("seeds_to_points", [C.c_void_p, C.c_size_t, C.c_void_p], seeds.ctypes.data_as(C.c_void_p), seeds.size,
                   out.ctypes.data_as(C.c_void_p))
        return out[: seeds.size].copy()

    def naive_propagate(self, pts, T_world_frame, reset_map):
        pts = np.ascontiguousarray(pts, dtype=DEPTH_POINT_DTYPE)
        T = _arr(T_world_frame, np.float64)
        self._call("naive_propagate", [C.c_void_p, C.c_size_t, C.POINTER(C.c_double), C.c_int],
                   pts.ctypes.data_as(C.c_void_p), pts.size, _ptr(T, C.c_double), int(reset_map))

    def map_clean(self, var_thr, age_thr, rho_max, rho_min):
        self._call("map_clean", [C.c_double] * 4, var_thr, age_thr, rho_max, rho_min)

    def map_regularize(self):
        self._call("map_regularize", [])

    def map_download(self):
        out = np.zeros(self.W * self.H, DEPTH_POINT_DTYPE)
        n = C.c_size_t(out.size)
        self._call("map_download", [C.c_void_p, C.POINTER(C.c_size_t)], out.ctypes.data_as(C.c_void_p), C.byref(n))
        return out[: n.value].copy()

    def mapping_at_time(self, ex, ey, et, pose_t, poses):
        ex, ey, et, pt, ps = self._ev_args(ex, ey, et, pose_t, poses)
        ctr = (C.c_uint64 * 8)()
        self._call("mapping_at_time", self._EV_TYPES + [C.POINTER(C.c_uint64)],
                   _ptr(ex, C.c_uint16), _ptr(ey, C.c_uint16), _ptr(et, C.c_int64), ex.size,
                   _ptr(pt, C.c_int64), _ptr(ps, C.c_double), pt.size, ctr)
        return _mapping_counters(ctr)

    def mapping_reset(self):
        self._call("mapping_reset", [])

    # ---- tracking ----
    def track_srand(self, seed):
        self._call("track_srand", [C.c_uint], seed)

    def track_reset(self, ref_xyz, T_world_ref, T_world_cur_prior, ts_left):
        """ref_xyz is permuted IN PLACE (float32 n x 3), like the reference."""
        assert ref_xyz.dtype == np.float32 and ref_xyz.flags.c_contiguous
        Tr = _arr(T_world_ref, np.float64); Tc = _arr(T_world_cur_prior, np.float64)
        ts = None if ts_left is None else _arr(ts_left, np.uint8)
        return self._call("track_reset",
                          [C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_uint8)],
                          _ptr(ref_xyz, C.c_float), ref_xyz.shape[0], _ptr(Tr, C.c_double), _ptr(Tc, C.c_double),
                          _ptr(ts, C.c_uint8), ok=(0, 1))

    def track_solve(self, analytical=True):
        T = np.zeros(16, np.float64)
        st = LMStats()
        self._call("track_solve", [C.c_int, C.POINTER(C.c_double), C.POINTER(LMStats)],
                   int(analytical), _ptr(T, C.c_double), C.byref(st))
        return T.reshape(4, 4), dict(n_points=st.n_points, nfev=st.nfev, n_iter=st.n_iter)

    def track_get_negative_ts(self):
        n = self.W * self.H
        a = np.empty(n); b = np.empty(n); c = np.empty(n)
        self._call("track_get_negative_ts", [C.POINTER(C.c_double)] * 3,
                   _ptr(a, C.c_double), _ptr(b, C.c_double), _ptr(c, C.c_double))
        return a.reshape(self.H, self.W), b.reshape(self.H, self.W), c.reshape(self.H, self.W)

    # ---- device-resident staging (product only) ----
    def stage_ts_events(self, cam, x, y, t_ns, pol):
        x = _arr(x, np.uint16); y = _arr(y, np.uint16); t = _arr(t_ns, np.int64); p = _arr(pol, np.uint8)
        self._call("stage_ts_events",
                   [C.c_int, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.POINTER(C.c_int64), C.POINTER(C.c_uint8), C.c_size_t],
                   cam, _ptr(x, C.c_uint16), _ptr(y, C.c_uint16), _ptr(t, C.c_int64), _ptr(p, C.c_uint8), x.size)

    def run_ts_build(self, cam, t_sync_ns):
        self._call("run_ts_build", [C.c_int, C.c_int64], cam, int(t_sync_ns))

    def stage_mapping_inputs(self, ex, ey, et, pose_t, poses):
        ex, ey, et, pt, ps = self._ev_args(ex, ey, et, pose_t, poses)
        self._call("stage_mapping_inputs", self._EV_TYPES,
                   _ptr(ex, C.c_uint16), _ptr(ey, C.c_uint16), _ptr(et, C.c_int64), ex.size,
                   _ptr(pt, C.c_int64), _ptr(ps, C.c_double), pt.size)

    def run_mapping(self):
        self._call("run_mapping", [])

    def fetch_mapping_counters(self):
        ctr = (C.c_uint64 * 8)()
        self._call("fetch_mapping_counters", [C.POINTER(C.c_uint64)], ctr)
        return _mapping_counters(ctr)

    def sgbm_compute(self, left=None, right=None, num_disparities=48, block_size=11, P1=None, P2=None, disp12_max_diff=-1,
                     pre_filter_cap=0, uniqueness_ratio=11):
        """cv::StereoSGBM (MODE_SGBM, minDisparity 0) on the device; defaults = the reference's parameters.  left/right None:
        the observation pair that is on the device."""
        P1 = 8 * block_size * block_size if P1 is None else P1
        P2 = 32 * block_size * block_size if P2 is None else P2
        out = np.zeros((self.H, self.W), np.int16)
        lp = rp = None
        if left is not None:
            l = _arr(left, np.uint8); r = _arr(right, np.uint8)
            assert l.size == self.W * self.H and r.size == l.size
            lp, rp = _ptr(l, C.c_uint8), _ptr(r, C.c_uint8)
        self._call("sgbm_compute", [C.POINTER(C.c_uint8), C.POINTER(C.c_uint8)] + [C.c_int] * 7 + [C.POINTER(C.c_int16)],
                   lp, rp, int(num_disparities), int(block_size), int(P1), int(P2), int(disp12_max_diff), int(pre_filter_cap),
                   int(uniqueness_ratio), _ptr(out, C.c_int16))
        return out

    def init_from_disparity(self, disp16, ex, ey, T_world_left, min_points):
        """InitializationAtTime downstream of the SGM call: returns (number of SGM depth points, accepted)."""
        d = _arr(disp16, np.int16); x = _arr(ex, np.uint16); y = _arr(ey, np.uint16)
        T = np.ascontiguousarray(T_world_left, np.float64)
        assert d.size == self.W * self.H
        n = C.c_size_t(0); acc = C.c_int(0)
        self._call("init_from_disparity",
                   [C.POINTER(C.c_int16), C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.c_size_t, C.POINTER(C.c_double), C.c_size_t,
                    C.POINTER(C.c_size_t), C.POINTER(C.c_int)],
                   _ptr(d, C.c_int16), _ptr(x, C.c_uint16), _ptr(y, C.c_uint16), x.size, _ptr(T, C.c_double), int(min_points),
                   C.byref(n), C.byref(acc))
        return int(n.value), bool(acc.value)

    # ---- event windows read from the time-surface log (product only) ----
    def events_window_dev(self, cam, front, t_begin_ns, t_end_ns, budget, denoise, max_keep, ok=(0,)):
        """esvo_events_window_dev: returns (rc, size of the selection); rc in ok, else EsvoError."""
        n = C.c_size_t(0)
        rc = self._call("events_window_dev", [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_size_t, C.c_int, C.c_size_t, C.POINTER(C.c_size_t)],
                        int(cam), int(front), int(t_begin_ns), int(t_end_ns), int(budget), int(bool(denoise)), int(max_keep), C.byref(n), ok=ok)
        return rc, int(n.value)

    def events_lower_bound_dev(self, cam, front, t_ns, ok=(0,)):
        """esvo_events_lower_bound_dev: returns (rc, global push indices)."""
        t = _arr(t_ns, np.int64)
        out = np.zeros(t.size, np.int64)
        rc = self._call("events_lower_bound_dev", [C.c_int, C.c_int64, C.POINTER(C.c_int64), C.c_size_t, C.POINTER(C.c_int64)],
                        int(cam), int(front), _ptr(t, C.c_int64), t.size, _ptr(out, C.c_int64), ok=ok)
        return rc, out

    def events_selected_dev(self):
        """The last selection (x, y, t, newest first), read back through device buffers."""
        import torch
        cap = max(int(self.evw_cap) if hasattr(self, "evw_cap") else 0, 1)
        while True:
            x = torch.zeros(cap, dtype=torch.int16, device="cuda"); y = torch.zeros(cap, dtype=torch.int16, device="cuda")
            t = torch.zeros(cap, dtype=torch.int64, device="cuda")
            n = C.c_size_t(cap)
            rc = self._call("events_selected_dev", [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t)], C.c_void_p(x.data_ptr()),
                            C.c_void_p(y.data_ptr()), C.c_void_p(t.data_ptr()), C.byref(n), ok=(0, -4))
            if rc == 0:
                k = int(n.value)
                return (x[:k].cpu().numpy().view(np.uint16), y[:k].cpu().numpy().view(np.uint16), t[:k].cpu().numpy())
            cap = int(n.value); self.evw_cap = cap

    def mapping_at_time_selected_dev(self, pose_t, poses):
        pt = _arr(pose_t, np.int64); ps = _arr(poses, np.float64)
        ctr = (C.c_uint64 * 8)()
        self._call("mapping_at_time_selected_dev", [C.POINTER(C.c_int64), C.POINTER(C.c_double), C.c_size_t, C.POINTER(C.c_uint64)],
                   _ptr(pt, C.c_int64), _ptr(ps, C.c_double), pt.size, ctr)
        return _mapping_counters(ctr)

    def init_from_disparity_selected_dev(self, disp16, T_world_left, min_points):
        d = _arr(disp16, np.int16); T = np.ascontiguousarray(T_world_left, np.float64)
        assert d.size == self.W * self.H
        n = C.c_size_t(0); acc = C.c_int(0)
        self._call("init_from_disparity_selected_dev", [C.POINTER(C.c_int16), C.POINTER(C.c_double), C.c_size_t, C.POINTER(C.c_size_t),
                                                        C.POINTER(C.c_int)],
                   _ptr(d, C.c_int16), _ptr(T, C.c_double), int(min_points), C.byref(n), C.byref(acc))
        return int(n.value), bool(acc.value)

    def ts_set_unordered_input(self, cam, enable):
        self._call("ts_set_unordered_input", [C.c_int, C.c_int], int(cam), int(bool(enable)))

    def window_download(self, index):
        out = np.zeros(self.W * self.H, DEPTH_POINT_DTYPE)
        n = C.c_size_t(out.size)
        self._call("window_download", [C.c_int, C.c_void_p, C.POINTER(C.c_size_t)], int(index), out.ctypes.data_as(C.c_void_p), C.byref(n))
        return out[: n.value].copy()

    def set_pipeline_depth(self, depth):
        self._call("set_pipeline_depth", [C.c_int], int(depth))

    def results_begin(self):
        t = C.c_int64(-1)
        self._call("results_begin", [C.POINTER(C.c_int64)], C.byref(t))
        return t.value

    def results_end(self, ticket):
        if not hasattr(self, "_res_buf"):
            self._res_buf = np.zeros(self.W * self.H, DEPTH_POINT_DTYPE)
        out = self._res_buf
        n = C.c_size_t(out.size)
        ctr = (C.c_uint64 * 8)()
        self._call("results_end", [C.c_int64, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)],
                   int(ticket), out.ctypes.data_as(C.c_void_p), C.byref(n), ctr)
        return out[: n.value], _mapping_counters(ctr)

    def results_end_view(self, ticket):
        """Zero-copy esvo_results_end: a numpy view of the slot's pinned landing buffer (valid until the slot's next results_begin)."""
        ptr = C.c_void_p(); n = C.c_size_t(0); ctr = (C.c_uint64 * 8)()
        self._call("results_end_view", [C.c_int64, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)],
                   int(ticket), C.byref(ptr), C.byref(n), ctr)
        if n.value:
            buf = (C.c_char * (n.value * DEPTH_POINT_DTYPE.itemsize)).from_address(ptr.value)
            out = np.frombuffer(buf, dtype=DEPTH_POINT_DTYPE, count=n.value)
        else:
            out = np.zeros(0, DEPTH_POINT_DTYPE)
        return out, _mapping_counters(ctr)

    def sync(self):
        self._call("sync", [])

    def stream(self):
        f = self.L.fn("stream"); f.argtypes = [C.c_void_p]; f.restype = C.c_void_p
        return f(self.ctx)

    def launch_count(self):
        f = self.L.fn("launch_count"); f.argtypes = [C.c_void_p]; f.restype = C.c_uint64
        return int(f(self.ctx))


# ---------------------------------------------------------------- the chunk inflater (include/esvo_b200_inflate.h)
CODEC_BZ2, CODEC_LZ4 = 1, 2


class Chunk(C.Structure):
    _fields_ = [("src", C.c_void_p), ("src_size", C.c_uint64), ("dst", C.c_void_p), ("dst_size", C.c_uint64),
                ("codec", C.c_int32), ("status", C.c_int32)]


class Inflater:
    """esvo_inflater: compressed bag chunks inflated on a device; no esvo_ctx needed."""

    def __init__(self, lib: Library, device: int = 0, scratch_bytes: int = 1 << 30):
        self.lib, self.h = lib, C.c_void_p()
        f = lib.fn("inflater_create")
        f.argtypes = [C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]
        f.restype = C.c_int
        rc = f(device, scratch_bytes, C.byref(self.h))
        if rc != 0:
            raise EsvoError(rc, "esvo_inflater_create")

    def last_error(self) -> str:
        f = self.lib.fn("inflater_last_error")
        f.argtypes = [C.c_void_p]
        f.restype = C.c_char_p
        return f(self.h).decode()

    def inflate(self, chunks, ok=(0,)):
        """chunks: [(codec, src bytes, dst_size)] -> (return code, [status], [output bytes or None for a refused chunk])."""
        srcs = [np.frombuffer(s, np.uint8) if not isinstance(s, np.ndarray) else _arr(s, np.uint8).ravel() for _, s, _ in chunks]
        dsts = [np.empty(int(m), np.uint8) for _, _, m in chunks]
        arr = (Chunk * max(1, len(chunks)))()
        for k, ((codec, _, m), s, d) in enumerate(zip(chunks, srcs, dsts)):
            arr[k] = Chunk(s.ctypes.data if s.size else None, s.size, d.ctypes.data if d.size else None, int(m), codec, 0)
        f = self.lib.fn("inflate_chunks")
        f.argtypes = [C.c_void_p, C.POINTER(Chunk), C.c_int]
        f.restype = C.c_int
        rc = f(self.h, arr, len(chunks))
        if rc not in ok:
            raise EsvoError(rc, "esvo_inflate_chunks", self.last_error())
        st = [arr[k].status for k in range(len(chunks))]
        return rc, st, [d.tobytes() if s == 0 else None for d, s in zip(dsts, st)]

    def close(self):
        if self.h:
            f = self.lib.fn("inflater_destroy")
            f.argtypes = [C.c_void_p]
            f(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
