"""Loading a trained weight table into an oracle env: the checkpoint loader the reference lacks (SURVEY section 5).

The oracle hands out a pointer to an env's own table (lobo_theta); the table is written through it, memory_size doubles at
a time.  An env evaluated under a policy trained elsewhere -- env b of a shared policy -- is then
lobo_create(env_index0 + b) -> set_theta -> lobo_go_greedy -> lobo_set_backtest(1) -> lobo_run on b's day.
"""
import ctypes as C


def theta_view(L, h, table, M):
    """ctypes view (no copy) of table 0 = Q_A / 1 = Q_B of oracle env h; None when the agent has no such table"""
    p = L.lobo_theta(h, table)
    return (C.c_double * M).from_address(C.addressof(p.contents)) if p else None


def set_theta(L, h, table, values, M):
    """values: memory_size doubles (ctypes array or bytes-like) -> table `table` of oracle env h"""
    dst = theta_view(L, h, table, M)
    assert dst is not None, "the agent has no table %d" % table
    raw = bytes(values)
    assert len(raw) == 8 * M, (len(raw), 8 * M)
    C.memmove(dst, raw, 8 * M)
