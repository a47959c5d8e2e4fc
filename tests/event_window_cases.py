"""Case table of the event windows read from the time-surface log (include/esvo_b200.h: esvo_events_window_dev,
esvo_events_lower_bound_dev), and their host forms in numpy.

A case is a left event stream pushed into camera 0 in batches, and queries against it:
  * ("window", front, t_begin_ns, t_end_ns, budget, denoise, max_keep) -- the walk of frontend::selectCloseEvents /
    selectSGMEvents over the deque events[front:total], then createDenoisingMask + extractDenoisedEvents;
  * ("lower_bound", front, stamps) -- tools::EventBuffer_lower_bound over the same deque, as global push indices.
Streams are built deterministically.  expect() gives the host form's answer, or None where the resident log of the product
cannot answer (log model: LOG_CAP events, the oldest folded out when a push would overflow, keeping LOG_CAP / 4)."""
import functools

import numpy as np

W, H = 346, 260
LOG_CAP = 1 << 22
MAPPER_CAP, TRACKER_CAP = 3_000_000, 5_000_000
EPOCH = 1_600_000_000 * 10**9


# ---------------------------------------------------------------- host forms
def to_sec(t):
    """ros::Time::toSec() over an int64 array: sec + 1e-9 * nsec, product and sum rounded separately."""
    t = np.asarray(t, np.int64)
    s, n = np.divmod(t, 1_000_000_000)
    return s.astype(np.float64) + 1e-9 * n.astype(np.float64)


def from_sec(t):
    """ros::Time(double)."""
    sec = int(np.floor(t))
    nsec = int(np.round((t - sec) * 1e9))
    sec += nsec // 1_000_000_000
    return sec * 1_000_000_000 + nsec % 1_000_000_000


def t_begin_for(t_end_ns, window_s):
    """t_begin as dataTransferring computes it: fromSec(max(0, toSec(t_end) - window))."""
    return from_sec(max(0.0, float(to_sec([t_end_ns])[0]) - window_s))


def walk(secs, t_begin_ns, t_end_ns, budget):
    """selectCloseEvents / selectSGMEvents on a deque whose toSec() stamps are secs: indices into the deque, newest first."""
    v_end, v_begin = to_sec([t_end_ns, t_begin_ns])
    ev_end = int(np.searchsorted(secs, v_end, side="left"))
    ev_begin = int(np.searchsorted(secs, v_begin, side="left"))
    if ev_end == secs.size and ev_end != ev_begin and budget > 0:    # the one-past-the-end slot
        ev_end -= 1; budget -= 1
    n = min(budget, ev_end - ev_begin) if ev_end > ev_begin else 0
    return np.arange(ev_end, ev_end - n, -1, dtype=np.int64)


def mask_of(x, y):
    """createDenoisingMask: event map of the events with x < W, y < H, cv::medianBlur 3x3 (replicated borders)."""
    import cv2
    img = np.zeros((H, W), np.uint8)
    ok = (x < W) & (y < H)
    img[y[ok].astype(int), x[ok].astype(int)] = 255
    return cv2.medianBlur(img, 3)


def extract(x, y, mask, max_keep):
    """extractDenoisedEvents: the events whose mask value at the flat index y * W + x is 255, in order, at most max_keep.  A flat
    index past the image (undefined in the reference) is not kept."""
    flat = y.astype(np.int64) * W + x.astype(np.int64)
    inside = flat < W * H
    keep = np.zeros(x.size, bool)
    keep[inside] = mask.ravel()[flat[inside]] == 255
    return np.nonzero(keep)[0][:max_keep]


def neighbours_on(x, y):
    """How many of the 3x3 neighbours (borders replicated) of each event's pixel carry an event."""
    img = np.zeros((H, W), np.int32)
    ok = (x < W) & (y < H)
    img[y[ok].astype(int), x[ok].astype(int)] = 1
    p = np.pad(img, 1, mode="edge")
    cnt = sum(p[1 + dy: 1 + dy + H, 1 + dx: 1 + dx + W] for dy in (-1, 0, 1) for dx in (-1, 0, 1))
    return cnt


# ---------------------------------------------------------------- the resident log
def log_model(batches):
    """log_base (global index of the oldest resident event) after pushing batches of these sizes (ts.cu ts_make_room)."""
    base, n = 0, 0
    for b in batches:
        if n + b > LOG_CAP:
            keep = min(n, LOG_CAP // 4)
            base += n - keep; n = keep
        n += b
    return base


# ---------------------------------------------------------------- streams
def _ordered(rng, n, t0, step_max, xy=None, step_min=300):
    # stamps at least 300 ns apart: distinct doubles even at the epoch (1 ulp of 1.6e9 s is ~238 ns)
    t = t0 + np.cumsum(rng.integers(step_min, step_max + 1, n)).astype(np.int64)
    if xy is None:
        x = rng.integers(0, W, n).astype(np.uint16); y = rng.integers(0, H, n).astype(np.uint16)
    else:
        x, y = xy
    return x, y, t


def _clustered(rng, n, t0, step_max):
    """Events on a few short edges, so the median keeps some and drops others, plus stray events and hand-placed ones:
    (0, 0) alone (4 of 9 on at the corner), (W-1, H-1) with (W-2, H-2) (5 of 9 at the corner), x = W, y = H, 65535.
    Stamps step by 0 to step_max ns: runs of equal stamps."""
    cx = rng.integers(0, W, 12); cy = rng.integers(0, H, 12)
    k = rng.integers(0, 12, n)
    x = np.clip(cx[k] + rng.integers(-2, 3, n), 0, W - 1)
    y = np.clip(cy[k] + rng.integers(-1, 2, n), 0, H - 1)
    stray = rng.random(n) < 0.3
    x[stray] = rng.integers(0, W, stray.sum()); y[stray] = rng.integers(0, H, stray.sum())
    special = [(0, 0), (W - 1, H - 1), (W - 2, H - 2), (W, 10), (5, H), (65535, 3), (7, 65535), (W, H - 1), (W - 1, 0), (W - 1, 1),
               (0, 10), (0, 11), (0, 12)]                       # (W, 10) reads pixel (0, 11), which these switch on
    pos = n - 1 - rng.choice(900, len(special), replace=False)     # among the newest: every window newer than the stream walks them
    for p, (a, b) in zip(pos, special):
        x[p], y[p] = a, b
    t = t0 + np.cumsum(rng.integers(0, step_max + 1, n)).astype(np.int64)
    return x.astype(np.uint16), y.astype(np.uint16), t


def _windows_on(t, fronts, rng, pen=1000, half=0.001, n_ends=12):
    """BM and SGM windows at stamps inside the stream, at an event's own stamp, and newer than every event."""
    q = []
    ends = [int(t[-1]) + 1, int(t[-1]) + 10**9, int(t[-1])] + [int(t[i]) for i in rng.integers(0, t.size, n_ends)] + \
           [int(t[i]) + int(rng.integers(1, 1000)) for i in rng.integers(0, t.size, n_ends)]
    for front in fronts:
        for te in ends:
            q.append(("window", front, t_begin_for(te, 10 * half), te, pen, 1, pen))        # WORKING: BM, denoised
            q.append(("window", front, t_begin_for(te, 10 * half), te, pen, 0, pen))        # WORKING: BM, Denoising off
            q.append(("window", front, t_begin_for(te, 2 * half), te, pen + 1, 0, pen + 1))  # INITIALIZATION: SGM
    return q


@functools.lru_cache(maxsize=None)
def cases():
    out = {}
    rng = np.random.default_rng(11)
    # dense small stamps near 0: t_begin clamped at 0, the one-past-the-end rule, every budget edge
    x, y, t = _clustered(rng, 20_000, 1_000, 400)
    q = _windows_on(t, [0, 5000], rng)
    te = int(t[-1]) + 1
    for budget in (0, 1, 2, 10**6):
        q.append(("window", 0, t_begin_for(te, 0.01), te, budget, 1, budget))
    q.append(("window", 0, int(t[100]), int(t[100]), 1000, 1, 1000))       # empty window: t_begin == t_end
    q.append(("window", 0, int(t[0]) - 10, int(t[0]) - 5, 1000, 0, 1000))  # empty window before every event
    q.append(("window", 0, 0, te, 10**6, 1, 10**6))                        # the whole stream, budget larger than the window
    q.append(("window", 0, 0, int(t[0]), 10**6, 1, 10**6))                 # t_end at the oldest event
    q.append(("lower_bound", 0, [0, int(t[0]), int(t[5000]), int(t[-1]), int(t[-1]) + 1]))
    out["small_stamps"] = dict(x=x, y=y, t=t, batches=[7000, 7000, 6000], queries=q)
    # UNIX-epoch stamps whose neighbours share a double (1 ulp of 1.6e9 s is ~238 ns)
    x, y, t = _clustered(rng, 30_000, EPOCH + 123_456_789, 60)
    q = _windows_on(t, [0, 100], rng, n_ends=40)
    q.append(("lower_bound", 0, [int(t[i]) + d for i in rng.integers(0, t.size, 60) for d in (-1, 0, 1)]))
    out["epoch"] = dict(x=x, y=y, t=t, batches=[30_000], queries=q)
    # stamps a few seconds after zero, queried at the events' own stamps: there toSec()'s sum has a fine spacing (2^-52 s), and a
    # sum contracted into an FMA rounds ~1 stamp in 10 differently from the host's product-then-sum
    x, y, t = _clustered(rng, 30_000, 1_000_000_000 + 7, 90_000)
    q = _windows_on(t, [0], rng, n_ends=40)
    q.append(("lower_bound", 0, [int(t[i]) for i in rng.integers(0, t.size, 128)]))
    out["seconds"] = dict(x=x, y=y, t=t, batches=[30_000], queries=q)
    # an empty log
    e16 = np.zeros(0, np.uint16)
    out["empty"] = dict(x=e16, y=e16, t=np.zeros(0, np.int64), batches=[],
                        queries=[("window", 0, t_begin_for(10**9, 0.01), 10**9, 1000, 1, 1000), ("window", 0, 0, 0, 0, 0, 0),
                                 ("lower_bound", 0, [0, 10**9])])
    # the tracker's reset: its deque restarts at the push index of the reset, stamps before it answer `front`
    x, y, t = _ordered(rng, 50_000, EPOCH, 2000)
    r = 30_000
    out["tracker_reset"] = dict(x=x, y=y, t=t, batches=[30_000, 20_000], queries=[
        ("lower_bound", r, [int(t[1000]), int(t[r - 1]), int(t[r]), int(t[r + 500]), int(t[-1]) + 1]),
        ("lower_bound", 0, [int(t[1000]), int(t[r - 1])]),
        ("window", r, int(t[r - 100]), int(t[r + 800]), 2000, 0, 2000),
        ("window", r, int(t[r - 100]), int(t[-1]) + 1, 10**6, 0, 10**6)])
    # the mapper's 3e6 cap binding: the deque starts at total - 3e6 inside the resident log, and lower_bound(t_begin) falls
    # before it
    n = 3_500_000
    x, y, t = _ordered(rng, n, EPOCH, 400)
    f = n - MAPPER_CAP
    out["mapper_cap"] = dict(x=x, y=y, t=t, batches=[500_000] * 7, queries=[
        ("window", f, int(t[f - 1000]), int(t[f + 700]), 1000, 1, 1000),
        ("window", f, int(t[f - 1000]), int(t[f + 700]), 1000, 0, 1000),
        ("window", f, 0, int(t[f + 3]), 1000, 0, 1000),
        ("window", f, int(t[f - 10]), int(t[f]), 1000, 0, 1000),
        ("window", f, int(t[f - 1000]), int(t[-1]) + 1, 400_000, 0, 300_000),   # > 1024 compaction blocks, max_keep binding
        ("window", f, int(t[f - 1000]), int(t[-1]) + 1, 400_000, 1, 400_000),
        ("lower_bound", f, [0, int(t[f - 1]), int(t[f]), int(t[f + 1])])])
    # 7.5 M events: the oldest are folded out of the resident log.  Windows one event inside and one event past its boundary,
    # a window the budget ends inside it, and lower bounds of the tracker's (5e6) and the mapper's (3e6) deques around it.
    n = 7_500_000
    x, y, t = _ordered(rng, n, EPOCH, 1000)
    batches = [500_000] * 15
    B = log_model(batches)
    te = int(t[B + 900])
    out["evicted"] = dict(x=x, y=y, t=t, batches=batches, queries=[
        ("window", 0, int(t[B]), te, 10**4, 0, 10**4),          # lower_bound(t_begin) = B: answered
        ("window", 0, int(t[B - 1]), te, 10**4, 0, 10**4),      # lower_bound(t_begin) = B - 1, folded: refused
        ("window", 0, int(t[B - 1]), te, 901, 0, 901),          # the budget ends the walk at B: answered
        ("window", 0, int(t[B - 1]), te, 902, 0, 902),          # ... at B - 1: refused
        ("window", 0, int(t[B - 50]), int(t[B - 2]), 10, 0, 10),  # the whole window folded: refused
        ("window", n - MAPPER_CAP, int(t[B + 10]), te, 10**4, 1, 1000),
        ("lower_bound", n - TRACKER_CAP, [0, int(t[n - TRACKER_CAP]), int(t[B - 2]), int(t[B - 1]), int(t[B]), int(t[B + 1]), int(t[-1]) + 1]),
        ("lower_bound", n - MAPPER_CAP, [int(t[B - 1]), int(t[B]), int(t[B]) - 1])])
    return out


def stream_secs(case):
    return to_sec(case["t"])


def expect(case, query, secs=None):
    """The host form's answer to one query on the deque events[front:total], or None where the product's resident log cannot
    answer: ("window", selected global indices, walked global indices) / ("lower_bound", global indices)."""
    secs = stream_secs(case) if secs is None else secs
    B = log_model(case["batches"])
    total = case["t"].size
    if query[0] == "window":
        _, front, tb, te, budget, denoise, max_keep = query
        walked = front + walk(secs[front:], tb, te, budget)
        if not lower_bound_answerable(case, front, te, secs):
            return None                                      # lower_bound(t_end) among folded events, not pinned (events.cu)
        if walked.size and walked.min() < B:
            return None                                      # the walk leaves the resident log
        if not lower_bound_answerable(case, front, tb, secs):
            # lower_bound(t_begin) lies below the resident log: only a walk the budget ends is answered
            e_end = front + int(np.searchsorted(secs[front:], to_sec([te])[0]))
            if walked.size < (budget - 1 if e_end == total and budget > 0 else budget):
                return None
        x, y = case["x"][walked], case["y"][walked]
        sel = extract(x, y, mask_of(x, y), max_keep) if denoise else np.arange(min(walked.size, max_keep))
        return walked[sel], walked
    _, front, stamps = query
    out = []
    for s in stamps:
        i = front + int(np.searchsorted(secs[front:], to_sec([s])[0]))
        out.append(i)
    return np.array(out, np.int64)


def lower_bound_answerable(case, front, stamp, secs=None):
    """Whether the resident log (plus the newest folded stamp and the first stamp) pins lower_bound(stamp) (events.cu)."""
    secs = stream_secs(case) if secs is None else secs
    B = log_model(case["batches"])
    if front >= B:
        return True
    v = to_sec([stamp])[0]
    lo = int(np.searchsorted(secs[B:], v))
    return lo > 0 or secs[B - 1] < v or v <= secs[0]
