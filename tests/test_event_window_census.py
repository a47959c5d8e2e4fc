"""CPU: the case table of tests/test_gpu_event_windows.py (tests/event_window_cases.py) reaches every rule the device event
windows pin: the one-past-the-end slot and t_end inside the log, t_begin clamped at 0, an empty log, an empty window, budget 0
and a budget larger than the window, BM and SGM budgets, epoch stamps that share a double, events at x = W, y = H and 65535,
mask pixels with exactly 4 and 5 neighbours on (also on the border), windows answered and refused at the resident boundary,
the mapper's deque cap binding, the tracker's bounds past the resident log, and a front after a tracker reset."""
import numpy as np

import event_window_cases as ewc


def _census():
    hit = set()
    for name, case in ewc.cases().items():
        secs = ewc.stream_secs(case)
        t = case["t"]
        total = t.size
        B = ewc.log_model(case["batches"])
        if total == 0:
            hit.add("empty log")
        for q in case["queries"]:
            exp = ewc.expect(case, q, secs)
            if q[0] == "lower_bound":
                _, front, stamps = q
                if front > 0 and name == "tracker_reset":
                    full = np.searchsorted(secs, ewc.to_sec(stamps))
                    if (full < front).any():
                        hit.add("tracker reset front binds")
                for s in stamps:
                    ok = ewc.lower_bound_answerable(case, front, s, secs)
                    if front == total - ewc.TRACKER_CAP and front < B:
                        hit.add("tracker bound answered past the boundary" if ok else "tracker bound refused")
                    if name == "seconds" and s in t and s >= 10**9:
                        hit.add("lower bound at an event's own stamp, seconds > 0")
                    v = ewc.to_sec([s])[0]
                    if np.searchsorted(secs, v) != np.searchsorted(t, s):
                        hit.add("lower bound decided by a shared double")
                continue
            _, front, tb, te, budget, denoise, max_keep = q
            if exp is None:
                hit.add("window refused")
                continue
            sel, walked = exp
            hit.add("window answered past a fold" if B > 0 else "window answered")
            v_end = ewc.to_sec([te])[0]
            e_end = front + int(np.searchsorted(secs[front:], v_end))
            if total > 0 and walked.size:
                hit.add("one past the end" if e_end == total else "t_end inside the log")
            if tb == 0 and te > 0:
                hit.add("t_begin clamped at 0")
            if total > 0 and walked.size == 0:
                hit.add("empty window")
            if budget == 0:
                hit.add("budget 0")
            if 0 < walked.size < budget - 1:
                hit.add("budget larger than the window")
            hit.add("SGM budget" if budget == 1001 else "BM budget" if budget == 1000 else "other budget")
            if name == "mapper_cap" and int(np.searchsorted(secs, ewc.to_sec([tb])[0])) < front and walked.size and walked.min() == front + 1:
                hit.add("mapper cap binds")             # the walk stops at the deque's front, not at the stream's lower_bound
            if name == "evicted" and B > 0 and walked.size and walked.min() == B:
                hit.add("walk ends at the resident boundary")
            if name == "epoch":
                st = t[walked]
                if (np.diff(ewc.to_sec(st)) == 0).any() and (np.diff(st) != 0).any():
                    hit.add("walk over stamps that share a double")
            if denoise and walked.size:
                x, y = case["x"][walked], case["y"][walked]
                for tag, m in (("x = W", x == ewc.W), ("y = H", y == ewc.H), ("65535", (x == 65535) | (y == 65535))):
                    if m.any():
                        hit.add(tag)
                xk = case["x"][sel]
                if (xk == ewc.W).any():
                    hit.add("kept through the next row's first pixel")
                cnt = ewc.neighbours_on(x, y)
                ok = (x < ewc.W) & (y < ewc.H)
                c = cnt[y[ok].astype(int), x[ok].astype(int)]
                border = (x[ok] == 0) | (y[ok] == 0) | (x[ok] == ewc.W - 1) | (y[ok] == ewc.H - 1)
                for k in (4, 5):
                    if (c == k).any():
                        hit.add(f"{k} neighbours on")
                    if ((c == k) & border).any():
                        hit.add(f"{k} neighbours on at the border")
    return hit


def test_case_table_reaches_every_rule():
    hit = _census()
    need = {"empty log", "window answered", "window answered past a fold", "window refused", "one past the end",
            "t_end inside the log", "t_begin clamped at 0", "empty window", "budget 0", "budget larger than the window", "SGM budget",
            "BM budget", "lower bound decided by a shared double", "walk over stamps that share a double", "x = W", "y = H", "65535",
            "kept through the next row's first pixel", "4 neighbours on", "5 neighbours on", "4 neighbours on at the border",
            "5 neighbours on at the border", "walk ends at the resident boundary", "mapper cap binds", "tracker bound refused",
            "tracker bound answered past the boundary", "tracker reset front binds", "lower bound at an event's own stamp, seconds > 0"}
    assert need <= hit, sorted(need - hit)


def test_refusals_at_the_boundary_are_the_intended_ones():
    """In the 7.5 M-event stream: lower_bound(t_begin) at the first resident event is answered, one event earlier refused; a
    budget that ends the walk at the first resident event is answered, one more refused."""
    case = ewc.cases()["evicted"]
    got = [ewc.expect(case, q) is not None for q in case["queries"][:5]]
    assert got == [True, False, True, False, False]
