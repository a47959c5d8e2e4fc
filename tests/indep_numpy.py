"""Independent numpy/scipy re-derivation of the hot-path arithmetic, written from the REFERENCE sources only
(file:line cited per function) -- not from oracle/ and not from the CUDA kernels.  tests/test_indep_pins.py runs the
C++ oracle against these on the golden inputs, so that oracle and kernels are no longer checked only against a
restatement by the same reading (VERDICT r1, "what's weak" 1).  TEST INFRASTRUCTURE: plain f64 numpy, clarity over speed.
"""
import numpy as np


# ---- a5: tools::meanStdDev / normalizePatch (esvo_core/include/esvo_core/tools/utils.h:74-92),
#          EventBM::zncc_cost (esvo_core/src/core/EventBM.cpp:317-333)
def zncc_cost(pl, pr):
    pl = np.asarray(pl, np.float64); pr = np.asarray(pr, np.float64)
    n = pl.size

    def normalize(p):
        mean = p.sum() / n
        sub = p - mean
        sigma = np.sqrt((sub * sub).sum() / n) + 1e-6
        return (p - mean) / sigma
    return 0.5 * (1.0 - (normalize(pl) * normalize(pr)).sum() / n)


def bm_search(ts_l, ts_r, x1, dmin, dmax, wx, wy):
    """EventBM::epipolarSearching with step 1 (EventBM.cpp:170-226): integer-aligned patches centred on x1 = floor(rectified
    event) in the left and (x1.x - d, x1.y) in the right image; `cost <= min_cost` keeps the LATER disparity on ties (:198)."""
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    H, W = ts_l.shape
    x, y = int(x1[0]), int(x1[1])
    pl = ts_l[y - hy:y + hy + 1, x - hx:x + hx + 1]
    best, best_d = 1.0, None          # ZNCC_MAX_ = 1 (EventBM.h)
    for d in range(dmin, dmax + 1):
        x2 = x - d
        if x2 - hx < 1 or y - hy < 1 or x2 + hx >= W - 1 or y + hy >= H - 1:   # isValidPatch (:251-267)
            continue
        pr = ts_r[y - hy:y + hy + 1, x2 - hx:x2 + hx + 1]
        c = zncc_cost(pl, pr)
        if c <= best:
            best, best_d = c, d
    return best_d, best


# ---- a7: PerspectiveCamera::cam2World (esvo_core/src/container/CameraSystem.cpp:120-139): literal 4x4 inverse
def cam2world(P, x, inv_depth):
    z = 1.0 / inv_depth
    Pt = np.zeros((4, 4)); Pt[:3, :] = P; Pt[3, :] = [0, 0, 0, z]
    ps = z * np.linalg.inv(Pt) @ np.array([x[0], x[1], 1.0, 1.0])
    return ps[:3] / ps[3]


# ---- a8: DepthProblem::patchInterpolation (esvo_core/src/core/DepthProblem.cpp:193-262)
def patch_interpolation(img, loc, wx, wy):
    H, W = img.shape
    ulx = int(np.floor(loc[0])) - (wx - 1) // 2; uly = int(np.floor(loc[1])) - (wy - 1) // 2
    drx = int(np.floor(loc[0])) + (wx - 1) // 2; dry = int(np.floor(loc[1])) + (wy - 1) // 2
    if ulx < 0 or uly < 0 or drx >= W or dry >= H:
        return None
    ly, lx = int(np.floor(loc[1])), int(np.floor(loc[0]))
    q1 = (lx + 1) - loc[0]; q2 = loc[0] - lx; q3 = (ly + 1) - loc[1]; q4 = loc[1] - ly
    if uly + wy >= H or ulx + wx >= W:
        return None
    src = img[uly:uly + wy + 1, ulx:ulx + wx + 1].astype(np.float64)
    R = q1 * src[:, :wx] + q2 * src[:, 1:wx + 1]
    return q3 * R[:wy, :] + q4 * R[1:wy + 1, :]


# ---- a6/a7: DepthProblem::warping (:162-191) and operator() (:34-160) for LSnorm = Tdist, l2 and zncc
def depth_residual(rho, coor, T_left_virtual, Pl, Pr, ts_l, ts_r, wx, wy, nu, scale, norm="Tdist", info=None):
    """info (dict, optional) receives failed (the warp or the interpolation failed), trips (passes of the Tdist scale loop)
    and margin (the smallest |change / 0.05 - 1| the loop's 5 % test saw: where it is at rounding level, a last-bit
    difference of the residuals can change the number of passes and with it the whole vector)."""
    n = wx * wy
    if info is not None:
        info.update(failed=True, trips=0, margin=np.inf)
    H, W = ts_l.shape

    def fail():                                                                  # :43-59, :141-158
        if norm == "l2":
            return np.full(n, 255.0)
        if norm == "zncc":
            return np.full(n, 2 / np.sqrt(n))
        w = (nu + 1) / (nu + (255.0 / scale) ** 2)
        return np.full(n, np.sqrt(w) * 255.0)
    p_rv = cam2world(Pl, coor, rho)
    p_left = T_left_virtual[:3, :3] @ p_rv + T_left_virtual[:3, 3]
    h1 = Pl[:, :3] @ p_left + Pl[:, 3]; h2 = Pr[:, :3] @ p_left + Pr[:, 3]
    x1 = h1[:2] / h1[2]; x2 = h2[:2] / h2[2]
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    for xs in (x1, x2):
        if xs[0] < hx or xs[0] > W - hx or xs[1] < hy or xs[1] > H - hy:
            return fail()
    t1 = patch_interpolation(ts_l, x1, wx, wy)
    t2 = patch_interpolation(ts_r, x2, wx, wy) if t1 is not None else None
    if t1 is None or t2 is None:
        return fail()
    if info is not None:
        info["failed"] = False
    if norm == "l2":                                                             # :67-75
        return (t1 - t2).ravel()
    if norm == "zncc":                                                           # :76-87, tools::meanStdDev (utils.h:74-82)
        def standardise(t):
            mu = t.sum() / n
            sigma = np.sqrt(((t - mu) ** 2).sum() / n) + 1e-6
            return (t - mu) / sigma
        return ((standardise(t1) - standardise(t2)) / np.sqrt(n)).ravel()
    r = (t1 - t2).ravel(); r2 = r * r
    s1, s2, first = scale * scale, -1.0, True
    while first or abs(s2 - s1) / s1 > 0.05:                                    # :96
        if not first:
            s1 = s2
        nz = r != 0
        with np.errstate(over="ignore", divide="ignore"):
            tot = float(np.sum(r2[nz] * (nu + 1) / (nu + r2[nz] / s1)))        # :112-114 (order of summation differs)
        if tot == 0:
            s2 = scale * scale
            break
        s2 = tot / n
        first = False
        if info is not None:
            info["trips"] += 1
            info["margin"] = min(info["margin"], abs(abs(s2 - s1) / s1 / 0.05 - 1.0))
    with np.errstate(over="ignore", divide="ignore"):
        w = (nu + 1) / (nu + r2 / s2)
    return np.sqrt(w) * r


# ---- a11: DepthPoint::update_studentT (esvo_core/src/container/DepthPoint.cpp:166-188)
def update_student_t(state, rho, s2, var, nu):
    """state = dict(rho, s2, nu, var, age); rho <= -1e-6 means 'new point'."""
    st = dict(state)
    if st["rho"] > -1e-6:
        nu_u = min(nu, st["nu"])
        rho_u = (s2 * st["rho"] + st["s2"] * rho) / (st["s2"] + s2)
        s2_u = (nu_u + (st["rho"] - rho) ** 2 / (st["s2"] + s2)) / (nu_u + 1) * (st["s2"] * s2) / (st["s2"] + s2)
        st.update(rho=rho_u, s2=s2_u, nu=nu_u + 1)
        st["var"] = st["nu"] / (st["nu"] - 2) * st["s2"]
        st["age"] += 1
    else:
        st.update(rho=rho, s2=s2, var=var, nu=nu)
    return st


# ---- a12: DepthFusion::propagate_one_point (esvo_core/src/core/DepthFusion.cpp:18-68), Tdist branch
def propagate_point(p_cam, s2, nu, T_prop_prior, Pl, W, H):
    p = T_prop_prior[:3, :3] @ p_cam + T_prop_prior[:3, 3]
    h = Pl[:, :3] @ p + Pl[:, 3]
    x = h[:2] / h[2]
    if x[0] < 0 or x[0] >= W or x[1] < 0 or x[1] >= H:        # boundaryCheck (DepthFusion.cpp:194-199)
        return None
    rho = 1.0 / p[2]
    den = T_prop_prior[2, :2] @ p_cam[:2] + T_prop_prior[2, 3]
    den /= p_cam[2]
    den += T_prop_prior[2, 2]
    J = T_prop_prior[2, 2] / den ** 2
    s2p = J * J * s2
    return dict(row=int(np.floor(x[1])), col=int(np.floor(x[0])), x=x, rho=rho, s2=s2p, nu=nu, var=nu / (nu - 2) * s2p, p_cam=p)


# ---- tools::cayley2rot (esvo_core/src/tools/cayley.cpp:4-21)
def cayley2rot(c):
    c1, c2, c3 = c
    k = 1 + c1 * c1 + c2 * c2 + c3 * c3
    R = np.array([[1 + c1 * c1 - c2 * c2 - c3 * c3, 2 * (c1 * c2 - c3), 2 * (c1 * c3 + c2)],
                  [2 * (c1 * c2 + c3), 1 - c1 * c1 + c2 * c2 - c3 * c3, 2 * (c2 * c3 - c1)],
                  [2 * (c1 * c3 - c2), 2 * (c2 * c3 + c1), 1 - c1 * c1 - c2 * c2 + c3 * c3]])
    return R / k


# ---- RegProblemLM::computeJ_G (esvo_core/src/core/RegProblemLM.cpp:271-320), general x
def compute_J_G(x):
    c1, c2, c3 = x[:3]
    k = 1 + c1 ** 2 + c2 ** 2 + c3 ** 2; k2 = k * k
    A1 = np.array([[2 * c1 / k - 2 * c1 * (1 + c1 ** 2 - c2 ** 2 - c3 ** 2) / k2, -2 * c2 / k - 2 * c2 * (1 + c1 ** 2 - c2 ** 2 - c3 ** 2) / k2,
                    -2 * c3 / k - 2 * c3 * (1 + c1 ** 2 - c2 ** 2 - c3 ** 2) / k2],
                   [2 * c2 / k - 4 * c1 * (c1 * c2 + c3) / k2, 2 * c1 / k - 4 * c2 * (c1 * c2 + c3) / k2, 2 / k - 4 * c3 * (c1 * c2 + c3) / k2],
                   [2 * c3 / k - 4 * c1 * (c1 * c3 - c2) / k2, -2 / k + 4 * c2 * (c1 * c3 - c2) / k2, 2 * c1 / k - 4 * c3 * (c1 * c3 - c2) / k2]])
    A2 = np.array([[2 * c2 / k - 4 * c1 * (c1 * c2 - c3) / k2, 2 * c1 / k - 4 * c2 * (c1 * c2 - c3) / k2, -2 / k - 4 * c3 * (c1 * c2 - c3) / k2],
                   [-2 * c1 / k - 2 * c1 * (1 - c1 ** 2 + c2 ** 2 - c3 ** 2) / k2, 2 * c2 / k - 2 * c2 * (1 - c1 ** 2 + c2 ** 2 - c3 ** 2) / k2,
                    -2 * c3 / k - 2 * c3 * (1 - c1 ** 2 + c2 ** 2 - c3 ** 2) / k2],
                   [2 / k - 4 * c1 * (c1 + c2 * c3) / k2, 2 * c3 / k - 4 * c2 * (c1 + c2 * c3) / k2, 2 * c2 / k - 4 * c3 * (c1 + c2 * c3) / k2]])
    A3 = np.array([[2 * c3 / k - 4 * c1 * (c2 + c1 * c3) / k2, 2 / k - 4 * c2 * (c2 + c1 * c3) / k2, 2 * c1 / k - 4 * c3 * (c2 + c1 * c3) / k2],
                   [-2 / k - 4 * c1 * (c2 * c3 - c1) / k2, 2 * c3 / k - 4 * c2 * (c2 * c3 - c1) / k2, 2 * c2 / k - 4 * c3 * (c2 * c3 - c1) / k2],
                   [-2 * c1 / k - 2 * c1 * (1 - c1 ** 2 - c2 ** 2 + c3 ** 2) / k2, -2 * c2 / k - 2 * c2 * (1 - c1 ** 2 - c2 ** 2 + c3 ** 2) / k2,
                    2 * c3 / k - 2 * c3 * (1 - c1 ** 2 - c2 ** 2 + c3 ** 2) / k2]])
    J = np.zeros((12, 6))
    J[0:3, 0:3] = A1; J[3:6, 0:3] = A2; J[6:9, 0:3] = A3; J[9:12, 3:6] = np.eye(3)
    return J


def bilinear_1x1(img, loc):
    """RegProblemLM::patchInterpolation (RegProblemLM.cpp:418-487) for a 1x1 patch: value at a sub-pixel location."""
    H, W = img.shape
    lx, ly = int(np.floor(loc[0])), int(np.floor(loc[1]))
    if lx < 0 or ly < 0 or lx >= W or ly >= H or ly + 1 >= H or lx + 1 >= W:
        return None
    q1 = (lx + 1) - loc[0]; q2 = loc[0] - lx; q3 = (ly + 1) - loc[1]; q4 = loc[1] - ly
    s = img[ly:ly + 2, lx:lx + 2].astype(np.float64)
    R = q1 * s[:, 0] + q2 * s[:, 1]
    return q3 * R[0] + q4 * R[1]


def track_reproject(p, T, Pl, mask):
    """RegProblemLM::reprojection + isValidPatch for wx = wy = 1 (RegProblemLM.cpp:380-416)."""
    H, W = mask.shape
    pl = T[:3, :3] @ p + T[:3, 3]
    h = Pl[:, :3] @ pl + Pl[:, 3]
    x = h[:2] / h[2]
    if x[0] < 0 or x[0] > W - 1 or x[1] < 0 or x[1] > H - 1:
        return None
    if mask[int(x[1]), int(x[0])] < 125:
        return None
    return x


def warping_transformation(R_, t_, x):
    """RegProblemLM::getWarpingTransformation (RegProblemLM.cpp:322-346)."""
    dR = cayley2rot(x[:3])
    U, _, Vt = np.linalg.svd(R_.T @ dR.T)
    Rcr = U @ Vt
    T = np.eye(4); T[:3, :3] = Rcr; T[:3, 3] = -Rcr @ (x[3:] + dR @ t_)
    return T


def track_residuals(x, pts, R_, t_, Pl, mask, ts_neg, huber):
    """RegProblemLM::operator() + thread (RegProblemLM.cpp:91-176), 1x1 patches, LSnorm Huber (huber=None: l2)."""
    T = warping_transformation(R_, t_, x)
    out = np.empty(len(pts))
    for i, p in enumerate(pts):
        xs = track_reproject(p, T, Pl, mask)
        r = 255.0
        if xs is not None:
            v = bilinear_1x1(ts_neg, xs)
            if v is not None:
                r = v
        if huber is not None:
            w = huber / r if r > huber else 1.0
            out[i] = np.sqrt(w) * r
        else:
            out[i] = r
    return out


def track_jacobian(pts, R_, t_, Pl, mask, d_du, d_dv):
    """RegProblemLM::df at x = 0 (RegProblemLM.cpp:178-269) with J_G_0 = computeJ_G(0)."""
    JG0 = compute_J_G(np.zeros(6))
    Jc = R_.T @ np.array([[1.0 / Pl[0, 0], 0], [0, 1.0 / Pl[1, 1]], [0, 0]])
    T = np.eye(4); T[:3, :3] = R_.T; T[:3, 3] = -R_.T @ t_
    blk = np.zeros((len(pts), 12))
    for i, p in enumerate(pts):
        xs = track_reproject(p, T, Pl, mask)
        if xs is None:
            continue
        gx, gy = bilinear_1x1(d_du, xs), bilinear_1x1(d_dv, xs)
        if gx is None or gy is None:
            continue
        g = np.array([gx / 8, gy / 8])
        dPi = np.zeros((2, 3))
        dPi[:, :2] = Pl[:2, :2] / p[2]
        z2 = p[2] ** 2
        dPi[0, 2] = -(Pl[0, 0] * p[0] + Pl[0, 1] * p[1] + Pl[0, 3]) / z2
        dPi[1, 2] = -(Pl[1, 0] * p[0] + Pl[1, 1] * p[1] + Pl[1, 3]) / z2
        dT = np.zeros((3, 12))
        dT[:, 0:3] = p[0] * np.eye(3); dT[:, 3:6] = p[1] * np.eye(3); dT[:, 6:9] = p[2] * np.eye(3); dT[:, 9:12] = np.eye(3)
        blk[i] = g @ dPi @ Jc @ dPi @ dT * p[2]
    return -blk @ JG0


# ---- event front-end of esvo_Mapping::dataTransferring (esvo_core/src/esvo_Mapping.cpp:536-603), host logic ----
def ros_to_sec(ns):
    """ros::Time::toSec(): sec + 1e-9 * nsec."""
    s, n = divmod(int(ns), 1000000000)
    return float(s) + 1e-9 * float(n)


def ros_from_sec(t):
    """ros::Time(double): sec = floor(t), nsec = round((t - sec) * 1e9), normalised."""
    sec = int(np.floor(t))
    nsec = int(np.round((t - sec) * 1e9))
    sec += nsec // 1000000000
    nsec %= 1000000000
    return sec * 1000000000 + nsec


def select_close_events(t_events, t_end_ns, half_slice, process_event_num):
    """Indices of the events dataTransferring selects (:562-575): walk back from lower_bound(t_end) until lower_bound(t_begin)
    or PROCESS_EVENT_NUM pushes.  When no event is at/after t_end the reference's first push reads the slot one past the newest
    event (deque::end()); that slot is skipped here but still counts against PROCESS_EVENT_NUM (include/esvo_b200/esvo_core.hpp)."""
    t_events = np.asarray(t_events, np.int64)
    secs = np.array([ros_to_sec(t) for t in t_events])                    # EventBuffer_lower_bound compares toSec() doubles (utils.h:50-55)
    t_begin_ns = ros_from_sec(max(0.0, ros_to_sec(t_end_ns) - 10 * half_slice))
    ev_end = int(np.searchsorted(secs, ros_to_sec(t_end_ns), side="left"))
    ev_begin = int(np.searchsorted(secs, ros_to_sec(t_begin_ns), side="left"))
    out, budget = [], process_event_num
    if ev_end == t_events.size and ev_end != ev_begin and budget > 0:
        ev_end -= 1; budget -= 1
    while ev_end != ev_begin and len(out) < budget:
        out.append(ev_end); ev_end -= 1
    return np.array(out, np.int64)


def select_sgm_events(t_events, t_end_ns, half_slice, process_event_num):
    """The INITIALIZATION branch of dataTransferring (:538-552): window 2 * BM_half_slice_thickness, `<=` on the count (one event
    more than PROCESS_EVENT_NUM); the one-past-the-end slot is skipped like in select_close_events."""
    t_events = np.asarray(t_events, np.int64)
    secs = np.array([ros_to_sec(t) for t in t_events])
    t_begin_ns = ros_from_sec(max(0.0, ros_to_sec(t_end_ns) - 2 * half_slice))
    ev_end = int(np.searchsorted(secs, ros_to_sec(t_end_ns), side="left"))
    ev_begin = int(np.searchsorted(secs, ros_to_sec(t_begin_ns), side="left"))
    out, budget = [], process_event_num + 1
    if ev_end == t_events.size and ev_end != ev_begin:
        ev_end -= 1; budget -= 1
    while ev_end != ev_begin and len(out) < budget:
        out.append(ev_end); ev_end -= 1
    return np.array(out, np.int64)


def sample_pose_stamps(t_end_ns, half_slice):
    """Virtual-view stamps of st_map_ (:585-599): t_begin, then t <- Time(t.toSec() + 0.05 * BM_half_slice_thickness) while <= t_end."""
    t_end = ros_to_sec(t_end_ns)
    t = ros_from_sec(max(0.0, t_end - 10 * half_slice))
    out = []
    while ros_to_sec(t) <= t_end:
        out.append(t)
        t = ros_from_sec(ros_to_sec(t) + 0.05 * half_slice)
    return np.array(out, np.int64)


def pack_point_cloud(p_cam, T_world_frame):
    """publishPointCloud (:909-953): p_world = R p_cam + t as pcl::PointXYZ (f32), DepthMap iteration order."""
    T = np.asarray(T_world_frame, float).reshape(4, 4)
    return (np.asarray(p_cam) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)


# ---- comparison modes of esvo_MVStereo: EventMatcher [26] (esvo_core/src/core/EventMatcher.cpp) ----
def em_zncc_cost(pl, pr):
    """EventMatcher::zncc_cost (:253-274): mean-free patches divided by (Frobenius norm + 1e-6)."""
    pl = np.asarray(pl, np.float64); pr = np.asarray(pr, np.float64)
    ls = pl - pl.mean(); rs = pr - pr.mean()
    ln = ls / (np.linalg.norm(ls) + 1e-6); rn = rs / (np.linalg.norm(rs) + 1e-6)
    return 0.5 * (1.0 - float((ln * rn).sum()))


def _patch_fail_reason(loc, wx, wy, W, H):
    """Which test of patch_interpolation rejects loc: "ul" (ulx / uly < 0), "dr" (drx >= W / dry >= H), or "far_y" /
    "far_x" (only uly + wy >= H / only ulx + wx >= W: the row / column the bilinear weights reach beyond the window), or
    "far_xy" (both)."""
    fx, fy = int(np.floor(loc[0])), int(np.floor(loc[1]))
    ulx, uly = fx - (wx - 1) // 2, fy - (wy - 1) // 2
    if ulx < 0 or uly < 0:
        return "ul"
    if fx + (wx - 1) // 2 >= W or fy + (wy - 1) // 2 >= H:
        return "dr"
    if uly + wy >= H:
        return "far_xy" if ulx + wx >= W else "far_y"
    return "far_x"


def event_slicing_for_em(t_left, t_low_ns, t_up_ns, slice_thickness):
    """esvo_MVStereo::eventSlicingForEM (esvo_MVStereo.cpp:1008-1040) over the time-ordered left events vEventsPtr_left_:
    numSlice = floor((t_up - t_low) / thickness); a slice runs from its first event to lower_bound(first stamp + thickness)
    INCLUSIVE (the iterator itself belongs to the slice; end() steps back one), the next one starts behind it.
    Returns (counts, median stamps)."""
    t_left = np.asarray(t_left, np.int64)
    secs = np.array([ros_to_sec(t) for t in t_left])
    num = int(np.floor((ros_to_sec(t_up_ns) - ros_to_sec(t_low_ns)) / slice_thickness))
    counts, med = [], []
    it = 0
    for _ in range(num):
        t_end = ros_to_sec(ros_from_sec(secs[it] + slice_thickness))
        it_end = int(np.searchsorted(secs, t_end, side="left"))
        if it_end == t_left.size:
            it_end -= 1
        n = it_end - it + 1
        counts.append(n); med.append(int(t_left[it + n // 2]))
        it = it_end + 1
        if it == t_left.size:
            break
    return np.array(counts, np.int32), np.array(med, np.int64)


def event_match(left, right, slice_counts, slice_poses, lut_l, lut_r, Pl, Pr, baseline, ts_l, ts_r, T_world_left,
                time_thr, epi_thr, ncc_thr, wx, wy, num_thread, info=None):
    """EventMatcher::match_all_HyperThread / match / match_an_event (:60-163,185-251).  left / right: dicts of x, y, t, p
    (right time-ordered).  Returns a list of dicts in the reference's thread-major order and the number of zncc evaluations.
    info (dict, optional) receives counts of the decisions taken: winners by (lane, pass) of a 32-wide scan from the window's
    first candidate, exact cost ties with the winner, the no-candidate-scored fallback, epipolar decisions exactly at their
    bounds, candidates exactly on a window bound, and the patch test that rejected a warp."""
    H, W = ts_l.shape
    tsl = ts_l.astype(np.float64); tsr = ts_r.astype(np.float64)
    # EventSlice::numEvents_ is a size_t filled from an int: a non-positive count adds no event to the slice loop
    slice_of = np.repeat(np.arange(len(slice_counts)), np.maximum(np.asarray(slice_counts, np.int64), 0))
    total = min(slice_of.size, left["x"].size)
    census = dict(winners=[], ties=0, fallback_accept=0, fallback_reject=0, epi_eq_accept=0, epi_ulp_reject=0, disp_zero_reject=0,
                  disp_ulp_accept=0, on_low=0, on_up=0, warp_fail=0, patch_fail_ul=0, patch_fail_dr=0, patch_fail_far_y=0,
                  patch_fail_far_x=0, patch_fail_far_xy=0, total=total, num_thread=num_thread)
    if info is not None:
        info.update(census)
        census = info
    r_secs = np.array([ros_to_sec(t) for t in right["t"]])
    T_left_world = np.linalg.inv(np.asarray(T_world_left, float).reshape(4, 4))
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    evals = 0

    def one(i):
        nonlocal evals
        te = ros_to_sec(left["t"][i])
        low = ros_to_sec(ros_from_sec(te - time_thr / 2)); up = ros_to_sec(ros_from_sec(te + time_thr / 2))
        b = int(np.searchsorted(r_secs, low, side="left")); e = int(np.searchsorted(r_secs, up, side="left"))
        cand = [j for j in range(b, e) if low <= r_secs[j] <= up and bool(right["p"][j]) == bool(left["p"][i])]     # temporal + polarity (:66-88)
        census["on_low"] += sum(r_secs[j] == low for j in cand)
        census["on_up"] += int(np.sum(r_secs[e:] == up))             # `<= up` would take them; lower_bound(up) never offers them
        if not cand:
            return None
        xl = lut_l[int(left["y"][i]), int(left["x"][i])]
        epi = []
        for j in cand:                                                                                               # epipolar (:93-108)
            xr = lut_r[int(right["y"][j]), int(right["x"][j])]
            dy = abs(xl[1] - xr[1])
            census["epi_eq_accept"] += bool(dy == epi_thr and xr[0] < xl[0])
            census["epi_ulp_reject"] += bool(dy == np.nextafter(epi_thr, np.inf) and xr[0] < xl[0])
            census["disp_zero_reject"] += bool(dy <= epi_thr and xr[0] == xl[0])
            census["disp_ulp_accept"] += bool(dy <= epi_thr and xr[0] == np.nextafter(xl[0], -np.inf))
            if dy <= epi_thr and xr[0] < xl[0]:
                epi.append((j, xr))
        if not epi:
            return None
        T_world_rv = np.asarray(slice_poses[slice_of[i]], float).reshape(4, 4)
        T_left_rv = T_left_world @ T_world_rv
        f = Pl[0, 0]
        min_cost, best, best_depth = 1.0, 0, 0.0
        costs = []
        for q, (j, xr) in enumerate(epi):                                                                            # motion check (:110-150)
            depth = baseline * f / (xl[0] - xr[0])
            p_rv = cam2world(Pl, xl, 1.0 / depth)
            p_left = T_left_rv[:3, :3] @ p_rv + T_left_rv[:3, 3]
            h1 = Pl[:, :3] @ p_left + Pl[:, 3]; h2 = Pr[:, :3] @ p_left + Pr[:, 3]
            x1 = h1[:2] / h1[2]; x2 = h2[:2] / h2[2]
            if any(xs[0] < hx or xs[0] > W - hx or xs[1] < hy or xs[1] > H - hy for xs in (x1, x2)):               # warping2 (:276-306)
                census["warp_fail"] += 1
                continue
            pa = patch_interpolation(tsl, x1, wx, wy)
            pb = patch_interpolation(tsr, x2, wx, wy) if pa is not None else None
            if pa is None or pb is None:
                census["patch_fail_" + _patch_fail_reason(x1 if pa is None else x2, wx, wy, W, H)] += 1
                continue
            cost = em_zncc_cost(pa, pb); evals += 1
            costs.append(cost)
            if cost < min_cost:
                min_cost, best, best_depth = cost, q, depth
        if min_cost < 1.0:
            census["ties"] += sum(c == min_cost for c in costs) - 1
            k = epi[best][0] - b
            census["winners"].append((k % 32, k // 32 + 1))
        elif min_cost <= ncc_thr:
            census["fallback_accept"] += 1
        else:
            census["fallback_reject"] += 1
        if min_cost > ncc_thr:
            return None
        with np.errstate(divide="ignore"):
            inv = np.float64(1.0) / np.float64(best_depth)
        return dict(i=i, j=epi[best][0], x_left=xl, x_right=epi[best][1], t_ns=int(left["t"][i]), T=T_world_rv, inv_depth=float(inv), cost=min_cost)

    out = []
    for tid in range(num_thread):
        for i in range(tid, total, num_thread):
            m = one(i)
            if m is not None:
                out.append(m)
    return out, evals


def vemp_to_points(matches, Pl, age_vis_threshold):
    """esvo_MVStereo::vEMP2vDP (esvo_MVStereo.cpp:1072-1097)."""
    out = []
    for m in matches:
        out.append(dict(row=int(np.floor(m["x_left"][1])), col=int(np.floor(m["x_left"][0])), x=m["x_left"], inv_depth=m["inv_depth"],
                        variance=1e-6, residual=m["cost"], age=int(age_vis_threshold), p_cam=cam2world(Pl, m["x_left"], m["inv_depth"]), T=m["T"]))
    return out


# ---- a1: TimeSurface::eventsCallback (esvo_time_surface/src/TimeSurface.cpp:403-425) ----
def events_callback_queue(ev):
    """ev: dict of x, y, t (ns), p in ARRIVAL order, any stamp order.  Returns the same dict shape holding, per arrival, the event
    the callback hands to insertEvent: events_.back() after the new event has been insertion-sorted into events_."""
    events = []                                                                           # events_
    out = []
    for e in zip(ev["x"].tolist(), ev["y"].tolist(), ev["t"].tolist(), ev["p"].tolist()):
        events.append(e)                                                                  # :412
        i = len(events) - 2                                                               # :413
        while i >= 0 and events[i][2] > e[2]:                                             # :414, strict: e goes after equal stamps
            events[i + 1] = events[i]
            i -= 1
        events[i + 1] = e                                                                 # :419
        out.append(events[-1])                                                            # :421 events_.back()
    # clearEventQueue (:427-435) erases from the FRONT of events_ once it holds more than 5 000 000 entries; back() is never removed
    a = np.array(out, dtype=np.int64).reshape(-1, 4)
    return dict(x=a[:, 0].astype(np.uint16), y=a[:, 1].astype(np.uint16), t=a[:, 2].copy(), p=a[:, 3].astype(np.uint8))


# ---- a1/a2: EventQueueMat (esvo_time_surface/include/esvo_time_surface/TimeSurface.h:28-96) and
#      TimeSurface::createTimeSurfaceAtTime (esvo_time_surface/src/TimeSurface.cpp:52-152); image ops by OpenCV itself
def _queue_walk(ev_effective, T_ns, decay_ms, W, H, ignore_polarity, queue_len):
    """insertEvent for every arrival (ev_effective: what eventsCallback queued, in arrival order), then getMostRecentEventBeforeT
    and the decayed value per pixel.  Returns [(y, x, value)] in raster order and the grid of the arrival number each came from."""
    x = np.asarray(ev_effective["x"], np.int64); y = np.asarray(ev_effective["y"], np.int64)
    t = np.asarray(ev_effective["t"], np.int64); p = np.asarray(ev_effective["p"])
    arrival = np.nonzero((x < W) & (y < H))[0]                                            # insideImage; the others are never queued
    pix = y[arrival] * W + x[arrival]
    order = np.argsort(pix, kind="stable")                                                # per pixel, arrivals in push_back order
    sp = pix[order]
    from_back = np.searchsorted(sp, sp, side="right") - 1 - np.arange(sp.size)            # 0 = the queue's back()
    queued = arrival[order]
    # pop_front beyond queueLen leaves the last queue_len arrivals; the reverse walk of getMostRecentEventBeforeT returns the one
    # nearest the back with ts < T, i.e. the largest arrival number among them
    ok = (from_back < queue_len) & (t[queued] < T_ns)
    best = np.full(W * H, -1, np.int64)
    np.maximum.at(best, sp[ok], queued[ok])
    decay_sec = decay_ms / 1000.0
    hits = []
    idx = np.full((H, W), -1, np.int64)
    for q in np.nonzero(best >= 0)[0].tolist():                                           # ascending = the loops of :65-67, y outer, x inner
        i = int(best[q])
        ti = int(t[i])
        if not ros_to_sec(ti) > 0:                                                        # :73
            continue
        d = int(T_ns) - ti                                                                # ros::Duration (integer ns), then toSec()
        dt = float(d // 1000000000) + 1e-9 * float(d % 1000000000)
        v = np.exp(-dt / decay_sec)
        if not ignore_polarity:
            v *= 1.0 if p[i] else -1.0
        hits.append((q // W, q % W, float(v)))
        idx[q // W, q % W] = i
    return hits, idx


def _to_mono8(m, ignore_polarity, median_blur_kernel_size):
    import cv2
    m = 255.0 * m if ignore_polarity else 255.0 * (m + 1.0) / 2.0                         # :123-126
    img = np.clip(np.rint(m), 0, 255).astype(np.uint8)                                    # convertTo(CV_8U): saturate_cast(cvRound), half to even
    if median_blur_kernel_size > 0:
        img = cv2.medianBlur(img, 2 * median_blur_kernel_size + 1)                        # :130-131
    return img


def time_surface_backward(ev, T_ns, decay_ms, W, H, ignore_polarity, median_blur_kernel_size, map1, map2, queue_len=20, info=None):
    """ev: dict of x, y, t (ns), p in ARRIVAL order -- for out-of-order stamps the output of events_callback_queue.
    Returns (raw mono8 before remap, published mono8 after remap); info["idx"]: arrival number behind every pixel, -1 if none."""
    import cv2
    hits, idx = _queue_walk(ev, T_ns, decay_ms, W, H, ignore_polarity, queue_len)
    m = np.zeros((H, W), np.float64)
    for y, x, v in hits:
        m[y, x] = v                                                                       # :82-83
    img = _to_mono8(m, ignore_polarity, median_blur_kernel_size)
    out = cv2.remap(img, map1, map2, cv2.INTER_LINEAR)                                    # :149
    if info is not None:
        info["idx"] = idx
    return img, out


def time_surface_forward(ev_effective, T_ns, decay_ms, W, H, ignore_polarity, median_blur_kernel_size, lut, queue_len=20, info=None):
    """FORWARD mode (TimeSurface.cpp:86-116): every raw pixel, in raster order, splats its value onto the four neighbours of its
    rectified point (lut: H x W x 2, precomputed_rectified_points_), each of the four sums clamped at 1 right away and never from
    below.  The published image is this map as mono8 after the median; there is no remap (:138-142).  info: idx grid, the number
    of clamps that fired and the smallest map value before conversion."""
    hits, idx = _queue_walk(ev_effective, T_ns, decay_ms, W, H, ignore_polarity, queue_len)
    lut = np.asarray(lut, np.float64).reshape(H, W, 2)
    m = np.zeros((H, W), np.float64)
    clamps = 0
    for y, x, e in hits:
        u, v = float(lut[y, x, 0]), float(lut[y, x, 1])
        if not (u >= 0 and v >= 0):                                                       # :90 (false for NaN)
            continue
        u_i, v_i = int(np.floor(u)), int(np.floor(v))                                     # :92-93, size_t
        if not (u_i + 1 < W and v_i + 1 < H):                                             # :95
            continue
        fu, fv = u - u_i, v - v_i
        fu1, fv1 = 1.0 - fu, 1.0 - fv
        m[v_i, u_i] += fu1 * fv1 * e                                                      # :101-104
        m[v_i, u_i + 1] += fu * fv1 * e
        m[v_i + 1, u_i] += fu1 * fv * e
        m[v_i + 1, u_i + 1] += fu * fv * e
        for yy, xx in ((v_i, u_i), (v_i, u_i + 1), (v_i + 1, u_i), (v_i + 1, u_i + 1)):  # :106-113
            if m[yy, xx] > 1:
                m[yy, xx] = 1
                clamps += 1
    if info is not None:
        info.update(idx=idx, clamps=clamps, min_map=float(m.min()))
    return _to_mono8(m, ignore_polarity, median_blur_kernel_size)


# ---- a4: EventBM::match_an_event / match_all_HyperThread / match (esvo_core/src/core/EventBM.cpp:80-168,269-315) ----
def event_bm_match_all(ev, ts_l, ts_r, lut_l, mask_l, pose_t, poses, wx, wy, dmin, dmax, step, thr, baseline, P00, num_thread,
                       updown=False):
    """ev: dict x, y, t of the events handed to createMatchProblem (left camera, raw pixels).  Returns the EventMatchPairs (dicts)
    in the reference's thread-major order and the number of zncc evaluations.  updown: bUpDownConfiguration_, the right camera
    below the left one -- the search walks up the column instead of left along the row (:148-151, :181-184)."""
    H, W = ts_l.shape
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    tsl = ts_l.astype(np.float64); tsr = ts_r.astype(np.float64)
    pose_sec = np.array([ros_to_sec(t) for t in pose_t])
    evals = 0

    def valid(x, y):                                                   # isValidPatch (:251-267)
        return not (x - hx < 1 or y - hy < 1 or x + hx >= W - 1 or y + hy >= H - 1)

    def search(x1, patch, start, end, sstep, state):                   # epipolarSearching (:170-226)
        nonlocal evals
        costs = {}
        d = start
        while d <= end:
            x2 = (x1[0], x1[1] - d) if updown else (x1[0] - d, x1[1])
            if not valid(*x2):
                costs[d] = 1.0
            else:
                c = zncc_cost(patch, tsr[x2[1] - hy:x2[1] + hy + 1, x2[0] - hx:x2[0] + hx + 1])
                evals += 1
                costs[d] = c
                if c <= state["min"]:
                    state.update(min=c, bx=x2, bd=d)
            d += sstep
        if sstep > 1:
            lo, hi = state["bd"] - sstep, state["bd"] + sstep
            return lo in costs and hi in costs and costs[lo] < 1.0 and costs[hi] < 1.0 and state["min"] < thr
        return state["min"] < thr

    def one(i):
        xr = lut_l[int(ev["y"][i]), int(ev["x"][i])]
        if xr[0] < 0 or xr[0] > W - 1 or xr[1] < 0 or xr[1] > H - 1:
            return None
        if mask_l[int(xr[1]), int(xr[0])] <= 125:                      # Eigen's (double) index: truncation
            return None
        x1 = (int(np.floor(xr[0])), int(np.floor(xr[1])))
        if not valid(*x1):
            return None
        patch = tsl[x1[1] - hy:x1[1] + hy + 1, x1[0] - hx:x1[0] + hx + 1]
        if (patch < 1).sum() > 0.95 * patch.size:                      # low information-to-noise ratio (:104-109)
            return None
        st = dict(min=1.0, bx=(0, 0), bd=0)
        if not search(x1, patch, dmin, dmax, step, st):                # coarse
            return None
        # fine (:128-131): the start bestDisp - (step - 1) is a size_t; below 0 it wraps to a huge value and the loop is empty
        start = st["bd"] - (step - 1)
        if not search(x1, patch, start if start >= 0 else 2 ** 64 + start, st["bd"] + (step - 1), 1, st):
            return None
        if not st["min"] <= thr:
            return None
        disparity = float(x1[1] - st["bx"][1]) if updown else float(x1[0] - st["bx"][0])
        k = int(np.searchsorted(pose_sec, ros_to_sec(ev["t"][i]), side="left"))             # StampTransformationMap_lower_bound on toSec()
        if k == len(pose_t):
            return None
        depth = baseline * P00 / disparity
        return dict(i=i, x_left_raw=(float(ev["x"][i]), float(ev["y"][i])), x_left=xr, x_right=(float(st["bx"][0]), float(st["bx"][1])), t_ns=int(ev["t"][i]),
                    pose=k, inv_depth=1.0 / depth, cost=st["min"], disp=disparity)

    out = []
    n = len(ev["x"])
    for tid in range(num_thread):                                      # match (:300-315): thread tid takes events tid, tid + NT, ...
        for i in range(tid, n, num_thread):
            m = one(i)
            if m is not None:
                out.append(m)
    return out, evals
