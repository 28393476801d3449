#!/usr/bin/env python3
"""Write a clean md/tas CSV pair (the column layout of oracle/_ref/flow_csv, %.4f prices) for one trading day of any
venue, whose best bid crosses one chosen band boundary of that venue's tick table many times.

Prices are integers in units of 1e-4, so every level sits exactly on its band's grid; the levels of each side step along
that grid, so a ladder next to the boundary holds two tick sizes.  The best bid random-walks, pulled alternately to
either side of the boundary; spreads are 1..3 ticks.  Prints against the previous row's book land at bid-1, bid, ask and
ask+1 (at most four distinct prices per row: one row is one message).  Rows are evenly spaced, from before the venue's
open + 30 min to after its close - 30 min, with the last open row 10 ms before that guard (16:16 plus 40 ms is the Irish
close), so every day passes through Initialise's warm-up and ends at its own venue's close.

Test infrastructure, pure Python and seeded: used by tools/make_golden.py and the venue-day tests."""
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rl_markets_b200 import config  # noqa: E402

UNIT = 10000  # price units per currency unit


def _fmt_time(ms):
    return "%02d:%02d:%02d.%03d" % (ms // 3600000, ms // 60000 % 60, ms // 1000 % 60, ms % 1000)


class Grid:
    """The venue's tick table in price units."""

    def __init__(self, ticker):
        bands, self.open_ms, self.close_ms = config.venue_table(ticker)
        self.px = [int(round(p * UNIT)) for p, _ts in bands]
        self.ts = [int(round(ts * UNIT)) for _p, ts in bands]
        assert all(t > 0 for t in self.ts), ticker  # every tick size is a whole number of units

    def tick(self, p):
        """tick size of the band containing price p"""
        k = max(i for i in range(len(self.px)) if self.px[i] <= p)
        return self.ts[k]

    def up(self, p, n=1):
        for _ in range(n):
            p += self.tick(p)
        return p

    def down(self, p, n=1):
        for _ in range(n):
            p -= self.tick(p - 1)
        return p

    def top(self):
        """prices stay below the top band and the half tick under it"""
        return self.px[-1] - self.ts[-1]


def write_day(md_path, tas_path, ticker, boundary, seed, dt_ms=20000, thin=False, date=20100104):
    """Returns the number of depth rows written."""
    g = Grid(ticker)
    rnd = random.Random(seed)
    b = int(round(boundary * UNIT))
    assert b in g.px[1:-1], (ticker, boundary)
    open_lo, close_hi = g.open_ms + 30 * 60000, g.close_ms - 30 * 60000
    n_open = (close_hi - 10 - open_lo) // dt_ms + 1  # rows inside the session; the last one 10 ms before its end
    t_last = close_hi - 10
    t0 = t_last - (n_open - 1 + 40) * dt_ms
    n_rows = n_open + 40 + 40
    vol_lo, vol_hi = 100, 900
    bid = g.down(b, 6)
    spread = 1
    side, hold = 1, 0

    def fresh():  # thin: 1..20 lots, mostly a few, so that five levels often hold less than a position limit
        return 1 + int(19 * rnd.random() ** 3) if thin else rnd.randint(vol_lo, vol_hi)

    ask_v = [fresh() for _ in range(5)]
    bid_v = [fresh() for _ in range(5)]
    md = ["date,time,ap1,ap2,ap3,ap4,ap5,av1,av2,av3,av4,av5,bp1,bp2,bp3,bp4,bp5,bv1,bv2,bv3,bv4,bv5"]
    tas = ["date,time,price,size"]
    prev = None
    for r in range(n_rows):
        t = t0 + r * dt_ms
        if prev is not None:  # prints against the previous row's book, stamped with this row's time
            pb, pa = prev
            agg = {}
            for _ in range(rnd.choice((0, 1, 1, 2, 3))):
                p = rnd.choice((g.down(pb), pb, pa, g.up(pa)))
                agg[p] = agg.get(p, 0) + rnd.randint(1, 30 if thin else 300)
            for p in sorted(agg):
                tas.append("%d,%s,%.4f,%d" % (date, _fmt_time(t), p / UNIT, agg[p]))
            # the walk: pulled toward a point a few ticks on the current side of the boundary
            hold -= 1
            if hold <= 0:
                side, hold = -side, rnd.randint(20, 60)
            target = g.up(b, 4) if side > 0 else g.down(b, 5)
            u = rnd.random()
            if u < 0.35:
                bid = g.up(bid) if bid < target else (g.down(bid) if bid > target else bid)
            elif u < 0.5:
                bid = g.up(bid)
            elif u < 0.65:
                bid = g.down(bid)
            if rnd.random() < 0.2:
                spread = rnd.randint(1, 3)
            ask_v = [fresh() if thin else max(vol_lo, min(vol_hi, v + rnd.randint(-40, 40))) for v in ask_v]
            bid_v = [fresh() if thin else max(vol_lo, min(vol_hi, v + rnd.randint(-40, 40))) for v in bid_v]
        ask = g.up(bid, spread)
        aps = [g.up(ask, l) for l in range(5)]
        bps = [g.down(bid, l) for l in range(5)]
        assert aps[-1] < g.top() and bps[-1] > 0, (ticker, aps, bps)
        md.append("%d,%s,%s,%s,%s,%s" % (date, _fmt_time(t), ",".join("%.4f" % (p / UNIT) for p in aps),
                                         ",".join(str(v) for v in ask_v), ",".join("%.4f" % (p / UNIT) for p in bps),
                                         ",".join(str(v) for v in bid_v)))
        prev = (bid, ask)
    with open(md_path, "w") as f:
        f.write("\n".join(md) + "\n")
    with open(tas_path, "w") as f:
        f.write("\n".join(tas) + "\n")
    return n_rows


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--ticker", required=True)
    ap.add_argument("--boundary", type=float, required=True)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--thin", action="store_true")
    ap.add_argument("--md", required=True)
    ap.add_argument("--tas", required=True)
    a = ap.parse_args()
    print(write_day(a.md, a.tas, a.ticker, a.boundary, a.seed, thin=a.thin))
