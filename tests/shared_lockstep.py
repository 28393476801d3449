"""dtheta of one shared-policy tick against an exact sum of the updates that went into it.

A shared-policy tick adds every stepping env's update into dtheta; the device does it with fp64 atomics, so the order of
each weight's sum is free and nothing else is (DESIGN section 4).  The oracle's contribution log (lobo_batch_log) lists
every addition as (table, feature, value), value being the exact double added.  For the k contributions c_i of a weight
and s = their correctly rounded sum (math.fsum, started from +0 as dtheta is):

  k = 0       dtheta is 0;
  k = 1 or 2  dtheta == s bitwise: any order of one or two additions rounds once;
  k >= 3      |dtheta - s| <= (gamma_{k-1} + u) * sum|c_i| * (1 + k u),   u = 2^-53,  gamma_n = n u / (1 - n u):
              the error of any order or tree of round-to-nearest additions (Higham, Accuracy and Stability of
              Numerical Algorithms, section 4.2) plus the rounding of s and of the computed sum|c_i|.

A weight is *sensitive* when its smallest |c_i| exceeds twice that tolerance (any nonzero |c_i| for k <= 2): a sum that
lost, doubled or misrouted one addition is then more than the tolerance away from s, so it cannot pass.
"""
import ctypes as C
import math

import numpy as np

U = 2.0 ** -53
CONTRIB = np.dtype([("table", "<i4"), ("feature", "<i4"), ("value", "<f8")])


def gamma(n):
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1.0 - n * U)


def bind(L):
    """argtypes of the batch oracle's log and counters (oracle/lob_oracle.h)"""
    L.lobo_batch_log.argtypes = [C.c_void_p, C.c_int]
    L.lobo_batch_log_entries.restype = C.c_void_p
    L.lobo_batch_log_entries.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.lobo_batch_sum_traces.restype = C.c_int64
    L.lobo_batch_sum_traces.argtypes = [C.c_void_p]
    L.lobo_batch_stats.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    return L


def log_entries(L, b):
    """The last lobo_batch_accumulate's contributions as a numpy array of CONTRIB (a copy)"""
    n = C.c_int64()
    p = L.lobo_batch_log_entries(b, C.byref(n))
    if n.value == 0:
        return np.zeros(0, dtype=CONTRIB)
    return np.frombuffer((C.c_char * (n.value * CONTRIB.itemsize)).from_address(p), dtype=CONTRIB).copy()


class Tally:
    """What the checks of a run saw: touched weights, sensitive weights, the largest k, the worst error / bound."""

    def __init__(self):
        self.touched = self.sensitive = self.max_k = 0
        self.worst = 0.0
        self.ticks = 0

    def add(self, r):
        self.ticks += 1
        self.touched += r["touched"]
        self.sensitive += r["sensitive"]
        self.max_k = max(self.max_k, r["max_k"])
        self.worst = max(self.worst, r["worst"])

    @property
    def fraction(self):
        return self.sensitive / self.touched if self.touched else 0.0

    def __repr__(self):
        return "max k %d, worst error/bound %.3g, sensitive %d of %d touched weights (%.3f) over %d ticks" % (
            self.max_k, self.worst, self.sensitive, self.touched, self.fraction, self.ticks)


def sums(log, M):
    """Per touched weight of a tick's log: flat index (table * M + feature), k, the correctly rounded sum s, the
    tolerance (0 where k <= 2: bitwise) and whether the weight is sensitive."""
    keys = log["table"].astype(np.int64) * M + log["feature"].astype(np.int64)
    order = np.argsort(keys, kind="stable")
    ks, vs = keys[order], log["value"][order]
    uniq, start, k = np.unique(ks, return_index=True, return_counts=True)
    s = np.empty(len(uniq))
    one, two, many = k == 1, k == 2, k >= 3
    s[one] = 0.0 + vs[start[one]]
    s[two] = (0.0 + vs[start[two]]) + vs[start[two] + 1]
    vl = vs.tolist()
    s[many] = [0.0 + math.fsum(vl[a:a + n]) for a, n in zip(start[many].tolist(), k[many].tolist())]
    if len(uniq) == 0:
        return uniq, k, s, s.copy(), np.zeros(0, bool)
    av = np.abs(vs)
    abs_sum = np.add.reduceat(av, start)
    min_abs = np.minimum.reduceat(av, start)
    tol = np.where(many, (gamma(k - 1) + U) * abs_sum * (1.0 + k * U), 0.0)
    sensitive = np.where(many, min_abs > 2.0 * tol, min_abs > 0)
    return uniq, k, s, tol, sensitive


def check(log, dev, M):
    """log: CONTRIB entries of one tick; dev: the dtheta to check, either a dense float64 array (table A then table B,
    n_tables * M values) or (flat indices, values) of its nonzero entries, flat index = table * M + feature, indices
    ascending.  Returns dict(touched, sensitive, max_k, worst, bad): bad lists (table, feature, k, dtheta, s, tolerance)
    of every weight that breaks its rule (k = 0 with a nonzero dtheta included)."""
    uniq, k, s, tol, sensitive = sums(log, M)
    if isinstance(dev, np.ndarray):
        d = dev[uniq]
        other = np.ones(len(dev), dtype=bool)
        other[uniq] = False
        stray = np.flatnonzero(other & (dev != 0))
        stray_vals = dev[stray]
    else:
        idx, vals = dev
        full = np.zeros(len(uniq))
        pos = np.searchsorted(uniq, idx)
        hit = (pos < len(uniq)) & (uniq[np.minimum(pos, max(len(uniq) - 1, 0))] == idx) if len(uniq) else np.zeros(len(idx), bool)
        full[pos[hit]] = vals[hit]
        d = full
        stray, stray_vals = idx[~hit], vals[~hit]
    bad = [(int(w // M), int(w % M), 0, float(v), 0.0, 0.0) for w, v in zip(stray, stray_vals)]
    if len(uniq) == 0:
        return {"touched": 0, "sensitive": 0, "max_k": 0, "worst": 0.0, "bad": bad}
    many = k >= 3
    err = np.abs(d - s)
    ok = np.where(many, err <= tol, d.view(np.uint64) == s.view(np.uint64))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(many & (tol > 0), err / tol, 0.0)
    nbad = int((~ok).sum())
    for i in np.flatnonzero(~ok)[:20]:
        bad.append((int(uniq[i] // M), int(uniq[i] % M), int(k[i]), float(d[i]), float(s[i]), float(tol[i])))
    if nbad > 20:
        bad.append(("and %d more" % (nbad - 20),))
    return {"touched": len(uniq), "sensitive": int(sensitive.sum()), "max_k": int(k.max()), "worst": float(ratio.max()),
            "bad": bad}


def mutate(log, dtheta, M, how, rng):
    """A copy of the dense dtheta as a sum that went wrong in one addition, at a sensitive weight with the most
    contributions: how = "drop" (one addition lost), "double" (one made twice) or "move" (one landed in the other
    table).  Each wrong sum is the correctly rounded sum of the wrong multiset -- the best any order could do."""
    keys = log["table"].astype(np.int64) * M + log["feature"].astype(np.int64)
    uniq, k, _s, _tol, sensitive = sums(log, M)
    assert sensitive.any(), "no sensitive weight to mutate"
    n_most = int(k[sensitive].max())
    w = int(uniq[sensitive & (k == n_most)][0])
    vals = log["value"][keys == w].tolist()
    c = vals[rng.integers(len(vals))]
    out = dtheta.copy()
    if how == "drop":
        rest = list(vals)
        rest.remove(c)
        out[w] = 0.0 + math.fsum(rest)
    elif how == "double":
        out[w] = 0.0 + math.fsum(vals + [c])
    elif how == "move":
        rest = list(vals)
        rest.remove(c)
        out[w] = 0.0 + math.fsum(rest)
        w2 = (w + M) % (2 * M)
        other = log["value"][keys == w2].tolist()
        out[w2] = 0.0 + math.fsum(other + [c])
    else:
        raise ValueError(how)
    return out, n_most
