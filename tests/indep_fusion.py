"""Independent Python re-derivation of the map-side CONTROL FLOW of the hot path, written from the reference sources only:
DepthFusion::update / fusion (esvo_core/src/core/DepthFusion.cpp:71-192) with its case analysis (create / compatible fuse /
occlusion / replace), SmartGrid::set / clean / getNeighbourhood (esvo_core/include/esvo_core/container/SmartGrid.h:222-243,
308-316,367-386) and DepthRegularization::apply (esvo_core/src/core/DepthRegularization.cpp:19-110).
tests/test_indep_pins.py runs the C++ oracle against it, so that the fusion case analysis, the element order and the
regularisation are no longer checked only against a restatement by the same reading.  TEST INFRASTRUCTURE: plain Python
objects, clarity over speed (a few thousand points).  The fusion arithmetic (propagate_one_point, DepthPoint::update / update_studentT, chiSquareTest / studentTCompatibleTest)
is restated here in scalar Python floats, in the order the reference writes each expression, for both norms; cam2World
comes from tests/indep_numpy.py.
"""
import copy
import math

import numpy as np

import indep_numpy as ind


DBL_MIN = 2.2250738585072014e-308


def fast_path(S, nu_u):
    """The guard of fold_apply's branch-free Student-t update (esvo_b200/csrc/fuse.cu): which updates take rcp_nr / div_nr."""
    return 1e-200 < S < 1e200 and 2.0 < nu_u < 1e15


def fast_path_arms(S, nu_u, s2_map, s2_prop, count):
    """Counts both arms of every condition of the fast-path guard (stats keys S_lo / S_hi / nu_le2 / nu_big / fast), and
    denormal scale inputs."""
    count("S_lo" if not S > 1e-200 else "S_ok_lo")
    count("S_hi" if not S < 1e200 else "S_ok_hi")
    count("nu_le2" if not nu_u > 2.0 else "nu_ok_lo")
    count("nu_big" if not nu_u < 1e15 else "nu_ok_hi")
    if nu_u == 2.0:
        count("nu_eq2")
    if 0 < s2_map < DBL_MIN or 0 < s2_prop < DBL_MIN:
        count("s2_denormal")
    count("fast" if fast_path(S, nu_u) else "slow")


class Pt:
    """container::DepthPoint (DepthPoint.cpp:7-35): Student-t and Gaussian fields side by side."""

    def __init__(self, row=0, col=0):
        self.row, self.col = int(row), int(col)
        self.x = np.array([col + 0.5, row + 0.5])
        self.rho, self.var, self.res, self.age = -1.0, 0.0, 0.0, 0
        self.s2, self.nu = 0.0, 0.0                 # never initialised by the reference's constructors; the oracle's choice
        self.p_cam = np.zeros(3)

    def valid(self, *thr):
        if not thr:
            return self.rho > -1e-6                                               # DepthPoint.cpp:215-218
        var_thr, age_thr, rmax, rmin = thr                                        # :220-231
        return self.rho > -1e-6 and self.age >= age_thr and self.var <= var_thr and self.rho <= rmax and self.rho >= rmin

    def update(self, rho, var, count=lambda k: None):                            # DepthPoint.cpp:145-164
        if self.rho > -1e-6:
            temp = self.rho
            self.rho = (self.var * rho + var * temp) / (self.var + var)
            temp = self.var
            self.var = (temp * var) / (temp + var)
        else:
            self.rho, self.var = rho, var
            count("new_point")
        if self.var < 1e-6:                                                       # boundVariance (:140-143)
            self.var = 1e-6
            return True
        return False

    def update_student_t(self, rho, s2, var, nu, count=lambda k: None):          # DepthPoint.cpp:166-188
        if self.rho > -1e-6:
            nu_u = min(nu, self.nu)
            S = self.s2 + s2
            fast_path_arms(S, nu_u, self.s2, s2, count)
            rho_u = (s2 * self.rho + self.s2 * rho) / (self.s2 + s2)
            d = self.rho - rho                                                    # pow(x, 2) is x * x under -O3
            s2_u = (nu_u + (d * d) / (self.s2 + s2)) / (nu_u + 1) * (self.s2 * s2) / (self.s2 + s2)
            self.rho, self.s2, self.nu = rho_u, s2_u, nu_u + 1
            self.var = self.nu / (self.nu - 2) * self.s2
            self.age += 1
            if fast_path(S, nu_u):
                count("fast_var_in" if 1e-200 < self.var < 1e200 else "fast_var_out")
        else:
            self.rho, self.s2, self.var, self.nu = rho, s2, var, nu
            count("new_point")

    def copy_from(self, o):                                                       # DepthPoint::copy (:233-245): all but row / col
        self.rho, self.var, self.s2, self.nu = o.rho, o.var, o.s2, o.nu
        self.x, self.p_cam, self.res, self.age = o.x.copy(), o.p_cam.copy(), o.res, o.age


class Grid:
    """container::SmartGrid<DepthPoint>: a pointer grid over an insertion-ordered element list."""

    def __init__(self, rows, cols):
        self.rows, self.cols = rows, cols
        self.cell = {}           # (row, col) -> element
        self.elements = []       # insertion order (_elements)

    def exists(self, r, c):
        return (r, c) in self.cell

    def set(self, r, c, value):                                                   # SmartGrid.h:308-316
        if (r, c) not in self.cell:
            e = Pt(r, c)
            self.elements.append(e)
            self.cell[(r, c)] = e
        self.cell[(r, c)].copy_from(value)

    def assign(self, r, c, value):
        """`dm->get(row, col) = dp_prop`: the implicit assignment copies row_ / col_ too (DepthFusion.cpp:186)."""
        e = self.cell[(r, c)]
        e.copy_from(value)
        e.row, e.col = value.row, value.col

    def clean(self, var_thr, age_thr, rmax, rmin):                                # SmartGrid.h:222-243
        keep = []
        for e in self.elements:
            if e.valid(var_thr, age_thr, rmax, rmin):
                keep.append(e)
            else:
                # the reference clears _grid[temp->row()][temp->col()], i.e. the cell the ELEMENT names, which a replacement
                # (assign) may have pointed elsewhere (a dangling pointer there); like oracle and kernels this restatement
                # erases the cell that really holds the element
                for k, v in list(self.cell.items()):
                    if v is e:
                        del self.cell[k]
        self.elements = keep

    def neighbourhood(self, row, col, radius):                                    # SmartGrid.h:367-386
        out = []
        # `for (int r = row - radius; r <= row + radius; r++)` with size_t row / radius: for row < radius the start wraps to a
        # negative int that the size_t comparison then sees as huge -- the loop body never runs; the same for the columns
        if row < radius or col < radius:
            return out
        for r in range(row - radius, row + radius + 1):
            for c in range(col - radius, col + radius + 1):
                if 0 <= r < self.rows and 0 <= c < self.cols and (r, c) in self.cell and self.cell[(r, c)].valid():
                    out.append(self.cell[(r, c)])
        return out


def _sqrt(v):
    """C's sqrt: NaN for a negative argument (math.sqrt raises)."""
    return math.sqrt(v) if not v < 0 else math.nan


def mul4(A, B):
    """T = A * B of two 4 x 4 poses, each entry summed from 0 over k in order (the oracle's `mul`, Eigen's scalar order)."""
    out = [[0.0] * 4 for _ in range(4)]
    for i in range(4):
        for j in range(4):
            acc = np.float64(0.0)
            for k in range(4):
                acc = acc + A[i][k] * B[k][j]
            out[i][j] = acc
    return out


def rigid_inverse(T):
    """kindr's Transformation::inverse(): [R^T | -R^T t]."""
    I = [[np.float64(0.0)] * 4 for _ in range(4)]
    for i in range(3):
        for j in range(3):
            I[i][j] = T[j][i]
    for i in range(3):
        acc = np.float64(0.0)
        for k in range(3):
            acc = acc + I[i][k] * T[k][3]
        I[i][3] = -acc
    I[3][3] = np.float64(1.0)
    return I


def _pose(T):
    T = np.asarray(T, np.float64).reshape(4, 4)
    return [[T[i, j] for j in range(4)] for i in range(4)]


def propagate(p, T, P, W, H, norm, count=lambda k: None, naive=False):
    """DepthFusion::propagate_one_point (:18-68) or naive_propagate_one_point (:290-327), scalar, in the reference's order.
    p: dict p_cam, s2, nu, var, res, age.  Returns the propagated Pt, or None where boundaryCheck fails (a NaN pixel index
    passes it, but its size_t coordinates then fail every per-pixel check: None too)."""
    pc = [np.float64(v) for v in p["p_cam"]]
    pp = [T[i][0] * pc[0] + T[i][1] * pc[1] + T[i][2] * pc[2] + T[i][3] for i in range(3)]
    h = [P[i][0] * pp[0] + P[i][1] * pp[1] + P[i][2] * pp[2] + P[i][3] for i in range(3)]     # world2Cam
    x, y = h[0] / h[2], h[1] / h[2]
    if x < 0 or x >= W or y < 0 or y >= H:                                        # boundaryCheck (:194-199)
        count("outside")
        return None
    if x != x or y != y:
        count("nan_reprojection")
        return None
    prop = Pt(math.floor(y), math.floor(x))
    prop.x = np.array([x, y])
    inv_depth = np.float64(1.0) / pp[2]
    den = T[2][0] * pc[0] + T[2][1] * pc[1] + T[2][3]
    den = den / pc[2]
    den = den + T[2][2]
    J = T[2][2] / (den * den)
    if naive or norm == "l2":
        if prop.update(inv_depth, J * J * np.float64(p["var"])):
            count("l2_floor_prop")
    else:
        s2, nu = J * J * np.float64(p["s2"]), np.float64(p["nu"])
        prop.update_student_t(inv_depth, s2, nu / (nu - 2) * s2, nu)
    if inv_depth <= -1e-6:
        count("behind")
    prop.p_cam = np.array(pp)
    prop.res, prop.age = np.float64(p["res"]), int(p["age"])
    return prop


def fuse_vector(grid, pts, T_world_frame, Pl, W, H, radius, stats=None, norm="Tdist"):
    """DepthFusion::update (:71-87) of one vector of points (dicts: p_cam, s2, nu, var, res, age, T_world_cam) into `grid`.
    norm: "Tdist" (also what the project runs for zncc, DESIGN.md deviation 8) or "l2".  Returns the number of fusions;
    stats (dict, optional) counts the branches taken: create, fuse, occluded, replace, keep, new_point, the arms of the
    fast-path guard (fast_path_arms), l2_floor_prop / l2_floor_fuse, compat_nan, outside, nan_reprojection, behind."""
    count = (lambda k: stats.__setitem__(k, stats.get(k, 0) + 1)) if stats is not None else (lambda k: None)
    P = [[np.float64(v) for v in row] for row in np.asarray(Pl, float)]
    T_frame_world = rigid_inverse(_pose(T_world_frame))
    n_fusion = 0
    with np.errstate(all="ignore"):
        for p in pts:
            T = mul4(T_frame_world, _pose(p["T_world_cam"]))
            prop = propagate(p, T, P, W, H, norm, count)
            if prop is None:
                continue
            if radius == 0:                                                                                  # :97-121
                cells = [(prop.row + dy, prop.col + dx) for dy in (0, 1) for dx in (0, 1)]
            else:
                cells = [(prop.row + dy, prop.col + dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
            for (r, c) in cells:
                if c < 0 or c >= W or r < 0 or r >= H:                                                       # size_t wrap = out of range
                    continue
                if not grid.exists(r, c):                                                                    # case 1 (:126-145)
                    nw = Pt(r, c)
                    if norm == "l2":
                        nw.update(prop.rho, prop.var)
                    else:
                        nw.update_student_t(prop.rho, prop.s2, prop.var, prop.nu)
                    nw.res, nw.age = prop.res, prop.age
                    nw.p_cam = ind.cam2world(Pl, nw.x, float(prop.rho))
                    grid.set(r, c, nw)
                    count("create")
                    continue
                cur = grid.cell[(r, c)]
                if norm == "l2":                                                                             # chiSquareTest (:205-218)
                    d2 = (prop.rho - cur.rho) * (prop.rho - cur.rho)
                    chi = d2 / prop.var + d2 / cur.var
                    compat = chi < 5.99
                else:                                                                                        # studentTCompatibleTest (:221-231)
                    s1, s2 = _sqrt(prop.var), _sqrt(cur.var)
                    diff = abs(prop.rho - cur.rho)
                    if s1 != s1 or s2 != s2:
                        count("compat_nan")
                    compat = diff < 2 * s1 or diff < 2 * s2
                if compat:                                                                                   # case 2.1 (:162-177)
                    if norm == "l2":
                        if cur.update(prop.rho, prop.var, count):
                            count("l2_floor_fuse")
                    else:
                        cur.update_student_t(prop.rho, prop.s2, prop.var, prop.nu, count)
                    cur.age += 1
                    cur.res = min(cur.res, prop.res)
                    cur.p_cam = ind.cam2world(Pl, cur.x, float(prop.rho))
                    n_fusion += 1
                    count("fuse")
                else:                                                                                        # case 2.2 (:178-188)
                    if cur.rho - 2 * _sqrt(cur.var) > prop.rho:
                        count("occluded")
                        continue
                    if prop.var < cur.var and prop.res < cur.res:
                        grid.assign(r, c, prop)
                        count("replace")
                    else:
                        count("keep")
    return n_fusion


def regularize(grid, radius, min_nb, min_close, literal=True, norm="Tdist"):
    """DepthRegularization::apply (:19-110), the Tdist branch or (norm="l2") the inverse-variance weighted mean of :53-61.
    Returns the new grid (dm = dmTmp).
    literal=True: exactly as written -- `dmTmp.set(it->row(), it->col(), *it)` and the neighbourhood are keyed by the coordinates
    the element NAMES, which a replacement in the fusion (case 2.2) may have copied from another pixel: such an element is merged
    into the cell it names and its own cell vanishes.  literal=False: keyed by the cell that holds the element (the oracle's and
    the kernels' documented choice, DESIGN.md deviation 7); the named coordinates stay data."""
    true_cell = {id(e): k for k, e in grid.cell.items()}
    tmp = Grid(grid.rows, grid.cols)
    for it in grid.elements:
        kr, kc = (it.row, it.col) if literal else true_cell[id(it)]
        tmp.set(kr, kc, it)
        new = tmp.cell[(kr, kc)]
        if not literal:
            new.row, new.col = it.row, it.col
        if not it.valid():
            continue
        nbs = grid.neighbourhood(kr, kc, radius)
        is_set = False
        if len(nbs) > min_nb:
            close = [q for q in nbs if q.valid() and (abs(it.rho - q.rho) < 2.0 * math.sqrt(it.var) or abs(it.rho - q.rho) < 2.0 * math.sqrt(q.var))]
            if len(close) > min_close and norm == "l2":
                tot = 0.0
                for q in close:
                    tot += 1.0 / q.var
                mean = 0.0
                for q in close:
                    mean += q.rho * (1.0 / q.var) / tot
                new.rho = mean
                is_set = True
            elif len(close) > min_close:
                nu_post, rho_post, s2_post = close[0].nu, close[0].rho, close[0].s2
                for q in close[1:]:
                    nu_p, rho_p, s2_p = nu_post, rho_post, s2_post
                    nu_post = min(nu_p, q.nu)
                    rho_post = (q.s2 * rho_p + s2_p * q.rho) / (q.s2 + s2_p)
                    d = rho_p - q.rho
                    s2_post = (nu_post + (d * d) / (s2_p + q.s2)) / (nu_post + 1) * (s2_p * q.s2) / (s2_p + q.s2)
                new.rho = rho_post
                is_set = True
        if not is_set:
            new.rho = -1.0
    return tmp


def naive_propagate_vector(grid, pts, T_world_frame, Pl, W, H, stats=None):
    """DepthFusion::naive_propagation (DepthFusion.cpp:232-288) with naive_propagate_one_point (:290-327): Gaussian propagation,
    the four pixels around the re-projection, an empty pixel takes the point, an occupied one keeps the closer estimate and is
    replaced only by a propagated point with a smaller residual.  pts: dicts p_cam, var, res, age, T_world_cam.  stats (dict,
    optional) counts the branches taken: create, nearer, replace, keep."""
    count = (lambda k: stats.__setitem__(k, stats.get(k, 0) + 1)) if stats is not None else (lambda k: None)
    T_frame_world = np.linalg.inv(np.asarray(T_world_frame, float).reshape(4, 4))
    for p in pts:
        T = T_frame_world @ np.asarray(p["T_world_cam"], float).reshape(4, 4)
        pc = np.asarray(p["p_cam"], float)
        pp = T[:3, :3] @ pc + T[:3, 3]
        h = Pl[:, :3] @ pp + Pl[:, 3]
        x = h[:2] / h[2]
        if x[0] < 0 or x[0] >= W or x[1] < 0 or x[1] >= H:
            continue
        prop = Pt(int(math.floor(x[1])), int(math.floor(x[0])))
        prop.x = x
        den = (T[2, :2] @ pc[:2] + T[2, 3]) / pc[2] + T[2, 2]
        J = T[2, 2] / den ** 2
        prop.rho, prop.var = 1.0 / pp[2], max(J * J * p["var"], 1e-6)      # DepthPoint::update on a fresh point + boundVariance (:140-164)
        prop.p_cam, prop.res, prop.age = pp, p["res"], p["age"]
        for dy in (0, 1):
            for dx in (0, 1):
                r, c = prop.row + dy, prop.col + dx
                if c >= W or r >= H:
                    continue
                if not grid.exists(r, c):                                   # case 1
                    nw = Pt(r, c)
                    nw.rho, nw.var = prop.rho, max(prop.var, 1e-6)
                    nw.res, nw.age = prop.res, prop.age
                    nw.p_cam = ind.cam2world(Pl, nw.x, prop.rho)
                    grid.set(r, c, nw)
                    count("create")
                else:                                                       # case 2
                    cur = grid.cell[(r, c)]
                    if cur.rho > prop.rho:
                        count("nearer")
                        continue
                    if prop.res < cur.res:
                        grid.assign(r, c, prop)
                        count("replace")
                    else:
                        count("keep")
