"""Scalar restatement of the Student-t scale iteration of DepthProblem::operator() (DepthProblem.cpp:89-135) in Python floats,
with the arm every evaluation takes reported.  TEST INFRASTRUCTURE, clarity over speed.

The loop runs twice on the same residual vector:
  * `scale_loop_seq`: the reference's statements in its order (one sequential sum over the pixels, `r^2 (nu+1) / (nu + r^2/s)`);
  * `scale_loop_dev`: the kernels' (esvo_b200/csrc/lm.cu, depth_residual_half and lm2_kernel phase B): lane l of a half warp
    owns pixels l, l+16, ..., a sum is an in-lane sum followed by the 8/4/2/1 xor tree; the grouped-reciprocal form above a
    scale of 1e-30, one reciprocal per pixel down to 1e-250, plain divisions below.  The Newton-refined reciprocals and the
    fused multiply-adds of the first two arms are written as plain IEEE operations (both are within 1 ulp of them), so above
    1e-250 this order is the kernels' only up to rounding; the division arm, where every subnormal step is decided, is exact.
Where the two orders reach different outcomes (exit kind or scale at exit), or a 5 % test is decided within 1e-12 of its
threshold, the evaluation is *rounding-decided*: its result depends on the last bits of the arithmetic, not on the algorithm.
"""
import math

import numpy as np

DENORM_MIN = 5e-324
# DBL_MAX * 2^-1074 = 2^-50 - 2^-103: r^2 / s overflows once s is below r^2 / DBL_MAX, i.e. below r^2 / 2^-50 subnormal steps.
RESET_UNIT = 2.0 ** -50
# The shortcut's guard (DESIGN.md deviation 4): gap * min r^2 >= RESET_GAP * N with gap = 0.95 N - (nu+1) nz = 0.95 N eps.
RESET_GAP = 2.0 ** -49
# Below this gap per pixel, r_min > 1e-6 alone no longer proves the reset and the kernels reduce the minimum: 2^-49 / 1e-12.
GAP_NO_TINY = RESET_GAP / 1e-12


def _div(a, b):
    """C's a / b for a >= 0 (b == 0 -> +inf, 0 / 0 -> nan)."""
    if b == 0.0:
        return math.inf if a > 0 else math.nan
    return a / b


def degenerate(nz, N, nu):
    """The regime test both guards start from: (nu+1) m / N below 0.95 with a relative margin of 1e-9."""
    return (nu + 1) * float(nz) < 0.95 * float(N) * (1.0 - 1e-9)


def shortcut_old(r, N, nu):
    """The guard of the parent commit: degenerate and every non-zero |r| > 1e-6."""
    nzr = [abs(v) for v in r if v != 0]
    return degenerate(len(nzr), N, nu) and min(nzr, default=1e300) > 1e-6


def shortcut_new(r, N, nu):
    """The fixed guard: degenerate and gap * min r^2 >= 2^-49 N (both kernels; lm2_kernel reads min r^2 from r_min > 1e-6
    where the gap alone suffices, which only ever declines more cases)."""
    nzr = [v for v in r if v != 0]
    if not degenerate(len(nzr), N, nu):
        return False
    gap = 0.95 * float(N) - (nu + 1) * float(len(nzr))
    a2min = min((v * v for v in nzr if v * v != 0), default=1e300)
    return gap * a2min >= RESET_GAP * float(N)


def scale_loop_seq(r, N, nu, scale):
    """DepthProblem.cpp:89-119 statement by statement.  Returns dict(kind, sc2, passes, margin, below30, below250, subnormal):
    kind is 'reset' (sum == 0, scale back to td_scale^2), 'converged' (5 % test passed at a normal scale) or 'stall' (5 % test
    passed at a subnormal scale)."""
    r2 = [v * v for v in r]
    s1, s2, first = scale * scale, -1.0, True
    out = dict(passes=0, margin=math.inf, below30=False, below250=False, subnormal=False)
    while first or abs(s2 - s1) / s1 > 0.05:
        if not first:
            s1 = s2
        out["below30"] |= s1 <= 1e-30
        out["below250"] |= s1 <= 1e-250
        out["subnormal"] |= s1 < 2.2250738585072014e-308
        tot = 0.0
        for v, q in zip(r, r2):
            if v != 0:
                tot += _div(q * (nu + 1), nu + _div(q, s1))
        out["passes"] += 1
        if tot == 0:
            return dict(out, kind="reset", sc2=scale * scale)
        s2 = tot / N
        first = False
        if s1 >= 2.2250738585072014e-308:          # subnormal steps are exact multiples of 2^-1074 in both orders
            out["margin"] = min(out["margin"], abs(abs(s2 - s1) / s1 / 0.05 - 1.0))
    return dict(out, kind="stall" if s2 < 2.2250738585072014e-308 else "converged", sc2=s2)


def _lanes(vals, S):
    return [[vals[l + 16 * s] if l + 16 * s < len(vals) else 0.0 for s in range(S)] for l in range(16)]


def _half_sum(v):
    v = list(v)
    for o in (8, 4, 2, 1):
        v = [v[l] + v[l ^ o] for l in range(16)]
    return v[0]


def _group_sum(a, nus):
    """irls_lane_sum: a/x + b/y = (a y + b x) / (x y) over groups of four, three, two, one slots."""
    acc, S = 0.0, len(a)
    B = S - S % 4
    for s in range(0, B, 4):
        d = [nus + a[s + k] for k in range(4)]
        p01, p23 = d[0] * d[1], d[2] * d[3]
        n01, n23 = a[s] * d[1] + a[s + 1] * d[0], a[s + 2] * d[3] + a[s + 3] * d[2]
        acc += (n01 * p23 + n23 * p01) * (1.0 / (p01 * p23))
    R = S % 4
    if R == 3:
        d0, d1, d2 = nus + a[B], nus + a[B + 1], nus + a[B + 2]
        p01 = d0 * d1
        acc += ((a[B] * d1 + a[B + 1] * d0) * d2 + a[B + 2] * p01) * (1.0 / (p01 * d2))
    elif R == 2:
        d0, d1 = nus + a[B], nus + a[B + 1]
        acc += (a[B] * d1 + a[B + 1] * d0) * (1.0 / (d0 * d1))
    elif R == 1:
        acc += a[B] * (1.0 / (nus + a[B]))
    return acc


def _tree_sum(t):
    u, S, w = list(t), len(t), 1
    while w < S:
        for s in range(0, S - w, 2 * w):
            u[s] += u[s + w]
        w *= 2
    return u[0]


def scale_loop_dev(r, N, nu, scale, div_ge=False):
    """The kernels' literal loop (no shortcut) in their order; same result dict as scale_loop_seq.  div_ge=True writes the
    division arm's 5 % test with >= instead of > (a planted mistake that util.DEPTH_CASES must catch)."""
    S = 7 if N <= 112 else 8
    lanes = _lanes([v * v for v in r], S)
    nu1, invN = nu + 1, 1.0 / N
    sc1, run = scale * scale, True
    out = dict(passes=0, margin=math.inf, below30=False, below250=False, subnormal=False)

    def step(tot, div_test):
        nonlocal sc1, run
        out["passes"] += 1
        if tot == 0:
            run = False
            return dict(out, kind="reset", sc2=scale * scale)
        sc2 = tot * invN
        ch = abs(sc2 - sc1)
        run = (ch / sc1 >= 0.05 if div_ge else ch / sc1 > 0.05) if div_test else ch > 0.05 * sc1
        if sc1 >= 2.2250738585072014e-308:
            out["margin"] = min(out["margin"], abs(ch / sc1 / 0.05 - 1.0))
        sc1 = sc2
        if not run:
            return dict(out, kind="stall" if sc2 < 2.2250738585072014e-308 else "converged", sc2=sc2)
        return None
    while run and sc1 > 1e-30:
        res = step(nu1 * sc1 * _half_sum([_group_sum(a, nu * sc1) for a in lanes]), False)
        if res:
            return res
    out["below30"] = True
    while run and sc1 > 1e-250:
        nus, c1 = nu * sc1, nu1 * sc1
        res = step(_half_sum([_tree_sum([(q * c1) * (1.0 / (nus + q)) for q in a]) for a in lanes]), False)
        if res:
            return res
    out["below250"] = True
    while True:
        out["subnormal"] |= sc1 < 2.2250738585072014e-308
        tot = []
        for a in lanes:
            acc = 0.0
            for q in a:
                if q != 0:
                    acc += q * _div(nu1, nu + _div(q, sc1))
            tot.append(acc)
        res = step(_half_sum(tot), True)
        if res:
            return res


def weights(r, sc2, nu):
    """DepthProblem.cpp:121-133: f_i = sqrt((nu+1) / (nu + r_i^2 / s)) r_i, and the kernels' path: 'reciprocal' (scale above
    1e-200) or 'division' (the exact statements, taken by the whole warp when either half's scale is not above 1e-200)."""
    f = [math.sqrt(_div(nu + 1, nu + _div(v * v, sc2))) * v for v in r]
    return f, ("reciprocal" if sc2 > 1e-200 else "division")


def evaluate(r, N, nu, scale):
    """One evaluation of the Student-t residual on the residual vector r (N entries, zeros included), with both loops."""
    seq = scale_loop_seq(r, N, nu, scale)
    nz = sum(1 for v in r if v != 0)
    old, new = shortcut_old(r, N, nu), shortcut_new(r, N, nu)
    dev = dict(kind="reset", sc2=scale * scale, passes=0, margin=math.inf, below30=False, below250=False, subnormal=False) \
        if new else scale_loop_dev(r, N, nu, scale)
    f, path = weights(r, seq["sc2"], nu)
    # a stall's scale is a count of subnormal steps, decided by their rounding; a converged scale may differ in its last bits
    decided = seq["kind"] == dev["kind"] and min(seq["margin"], dev["margin"]) > 1e-12 and \
        (seq["kind"] != "stall" or seq["sc2"] == dev["sc2"]) and (new or seq["passes"] == dev["passes"])
    return dict(nz=nz, N=N, c=(nu + 1) * nz / N, seq=seq, dev=dev, shortcut_old=old, shortcut_new=new, f=f, path=path,
                rounding_decided=not decided)


# ---- the warp and the patch interpolation of the kernels for T_left_virtual = identity (the case table's seeds) ----
def cam2world_device(Pl, x, y, rho):
    """cam2world_dev (lm.cu) in its order of operations."""
    z = 1.0 / rho
    return [(x - Pl[0][2] - Pl[0][3] / z) * z / Pl[0][0], (y - Pl[1][2] - Pl[1][3] / z) * z / Pl[1][1], z * (1.0 - Pl[2][3] / z)]


def _inverse4(m):
    t = [0.0] * 16
    t[0] = m[5]*m[10]*m[15] - m[5]*m[11]*m[14] - m[9]*m[6]*m[15] + m[9]*m[7]*m[14] + m[13]*m[6]*m[11] - m[13]*m[7]*m[10]
    t[4] = -m[4]*m[10]*m[15] + m[4]*m[11]*m[14] + m[8]*m[6]*m[15] - m[8]*m[7]*m[14] - m[12]*m[6]*m[11] + m[12]*m[7]*m[10]
    t[8] = m[4]*m[9]*m[15] - m[4]*m[11]*m[13] - m[8]*m[5]*m[15] + m[8]*m[7]*m[13] + m[12]*m[5]*m[11] - m[12]*m[7]*m[9]
    t[12] = -m[4]*m[9]*m[14] + m[4]*m[10]*m[13] + m[8]*m[5]*m[14] - m[8]*m[6]*m[13] - m[12]*m[5]*m[10] + m[12]*m[6]*m[9]
    t[1] = -m[1]*m[10]*m[15] + m[1]*m[11]*m[14] + m[9]*m[2]*m[15] - m[9]*m[3]*m[14] - m[13]*m[2]*m[11] + m[13]*m[3]*m[10]
    t[5] = m[0]*m[10]*m[15] - m[0]*m[11]*m[14] - m[8]*m[2]*m[15] + m[8]*m[3]*m[14] + m[12]*m[2]*m[11] - m[12]*m[3]*m[10]
    t[9] = -m[0]*m[9]*m[15] + m[0]*m[11]*m[13] + m[8]*m[1]*m[15] - m[8]*m[3]*m[13] - m[12]*m[1]*m[11] + m[12]*m[3]*m[9]
    t[13] = m[0]*m[9]*m[14] - m[0]*m[10]*m[13] - m[8]*m[1]*m[14] + m[8]*m[2]*m[13] + m[12]*m[1]*m[10] - m[12]*m[2]*m[9]
    t[2] = m[1]*m[6]*m[15] - m[1]*m[7]*m[14] - m[5]*m[2]*m[15] + m[5]*m[3]*m[14] + m[13]*m[2]*m[7] - m[13]*m[3]*m[6]
    t[6] = -m[0]*m[6]*m[15] + m[0]*m[7]*m[14] + m[4]*m[2]*m[15] - m[4]*m[3]*m[14] - m[12]*m[2]*m[7] + m[12]*m[3]*m[6]
    t[10] = m[0]*m[5]*m[15] - m[0]*m[7]*m[13] - m[4]*m[1]*m[15] + m[4]*m[3]*m[13] + m[12]*m[1]*m[7] - m[12]*m[3]*m[5]
    t[14] = -m[0]*m[5]*m[14] + m[0]*m[6]*m[13] + m[4]*m[1]*m[14] - m[4]*m[2]*m[13] - m[12]*m[1]*m[6] + m[12]*m[2]*m[5]
    t[3] = -m[1]*m[6]*m[11] + m[1]*m[7]*m[10] + m[5]*m[2]*m[11] - m[5]*m[3]*m[10] - m[9]*m[2]*m[7] + m[9]*m[3]*m[6]
    t[7] = m[0]*m[6]*m[11] - m[0]*m[7]*m[10] - m[4]*m[2]*m[11] + m[4]*m[3]*m[10] + m[8]*m[2]*m[7] - m[8]*m[3]*m[6]
    t[11] = -m[0]*m[5]*m[11] + m[0]*m[7]*m[9] + m[4]*m[1]*m[11] - m[4]*m[3]*m[9] - m[8]*m[1]*m[7] + m[8]*m[3]*m[5]
    t[15] = m[0]*m[5]*m[10] - m[0]*m[6]*m[9] - m[4]*m[1]*m[10] + m[4]*m[2]*m[9] + m[8]*m[1]*m[6] - m[8]*m[2]*m[5]
    det = 1.0 / (m[0] * t[0] + m[1] * t[4] + m[2] * t[8] + m[3] * t[12])
    return [v * det for v in t]


def cam2world_literal(Pl, x, y, rho):
    """PerspectiveCamera::cam2World (CameraSystem.cpp:120-139): the cofactor inverse of [P; 0 0 0 z]."""
    z = 1.0 / rho
    Pi = _inverse4([float(v) for v in np.asarray(Pl).ravel()] + [0.0, 0.0, 0.0, z])
    xs = [x, y, 1.0, 1.0]
    ps = []
    for i in range(4):
        s = 0.0
        for k in range(4):
            s += (z * Pi[i * 4 + k]) * xs[k]
        ps.append(s)
    return [ps[0] / ps[3], ps[1] / ps[3], ps[2] / ps[3]]


def project(P, p):
    h = [P[q][0] * p[0] + P[q][1] * p[1] + P[q][2] * p[2] + P[q][3] for q in range(3)]
    return h[0] / h[2], h[1] / h[2]


def residual_vector(tl, tr, Pl, Pr, x, y, rho, wx, wy, cam2world=cam2world_device):
    """t1 - t2 of the patch at inverse depth rho for a seed at (x, y) with T_left_virtual = identity, or None where the warp or
    the interpolation fails (DepthProblem.cpp:162-239, lm.cu's bounds)."""
    H, W = tl.shape
    hx, hy = (wx - 1) // 2, (wy - 1) // 2
    p = cam2world(Pl, x, y, rho)
    pts = [project(Pl, p), project(Pr, p)]
    for (u, v) in pts:
        if not (u == u and v == v) or u < hx or u > W - hx or v < hy or v > H - hy:
            return None
    taps = []
    for img, (u, v) in zip((tl, tr), pts):
        fu, fv = math.floor(u), math.floor(v)
        ulx, uly = fu - hx, fv - hy
        if ulx < 0 or uly < 0 or fu + hx >= W or fv + hy >= H or uly + wy >= H or ulx + wx >= W:
            return None
        q1, q2, q3, q4 = (fu + 1) - u, u - fu, (fv + 1) - v, v - fv
        t = []
        for py in range(wy):
            for px in range(wx):
                a00, a01 = float(img[uly + py, ulx + px]), float(img[uly + py, ulx + px + 1])
                a10, a11 = float(img[uly + py + 1, ulx + px]), float(img[uly + py + 1, ulx + px + 1])
                t.append(q3 * (q1 * a00 + q2 * a01) + q4 * (q1 * a10 + q2 * a11))
        taps.append(t)
    return [a - b for a, b in zip(*taps)]


def failed_value(nu, scale):
    q = 255.0 / scale
    return math.sqrt((nu + 1) / (nu + q * q)) * 255.0


def reset_batch(R, nu, scale, max_passes=40000):
    """The reference's loop (sequential sums, numpy.cumsum accumulates left to right) over a batch of residual vectors at once,
    rows of R (zeros are skipped as DepthProblem.cpp:112 skips them).  Returns (kind, sc2) arrays: kind 0 reset, 1 stall,
    2 converged."""
    R = np.asarray(R, np.float64)
    B, N = R.shape
    R2, nz = R * R, R != 0
    s1 = np.full(B, scale * scale)
    kind = np.full(B, -1)
    sc2 = np.zeros(B)
    live = np.ones(B, bool)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore", under="ignore"):
        for _ in range(max_passes):
            if not live.any():
                break
            idx = np.nonzero(live)[0]
            s = s1[idx][:, None]
            term = np.where(nz[idx], R2[idx] * (nu + 1) / (nu + R2[idx] / s), 0.0)
            tot = np.cumsum(term, axis=1)[:, -1]
            z = tot == 0
            kind[idx[z]] = 0
            sc2[idx[z]] = scale * scale
            s2 = tot / N
            done = ~z & ~(np.abs(s2 - s1[idx]) / s1[idx] > 0.05)
            kind[idx[done]] = np.where(s2[done] < 2.2250738585072014e-308, 1, 2)
            sc2[idx[done]] = s2[done]
            s1[idx] = s2
            live[idx[z | done]] = False
    assert not live.any()
    return kind, sc2
