"""config/example.yaml keys -> rlm_config (include/rlm.h).

Mirrors where and how the reference reads each key (SURVEY.md section 5), quirks
included:
  * learning.*            src/rl/agent.cpp:14-50, src/rl/state.cpp:22-24
  * policy.*              src/main.cpp:137-165 (eps/tau are read as *float*)
  * reward.*, state.lookback.*, market.*   src/environment/base.cpp:18-112
  * state.variables       src/environment/intraday.cpp:52-62
  * market.target_price.type is kept AS WRITTEN; the inverted selector of
    base.cpp:101-112 is applied inside the library (Appendix A1).
  * the fee key is upper-case TRANSACTION_FEE and unused (base.cpp:23, A12) -> ignored.
  * venue tick tables and trading hours: src/market/market.cpp:40-61,142-314 (all 14 venues).
"""
import ctypes as C

import yaml

from . import abi

HOUR, MINUTE = 3600000, 60000

# Tick-size tables of src/market/market.cpp:142-314, ascending (price from, tick size)
_EURONEXT = [(0.0, 0.001), (10.0, 0.005), (50.0, 0.01), (100.0, 0.05)]                       # :142-149
_NORDIC = [(0.0, 0.0001), (0.5, 0.0005), (1.0, 0.001), (2.0, 0.002), (5.0, 0.005), (10.0, 0.01), (50.0, 0.05),
           (100.0, 0.1), (500.0, 0.5), (1000.0, 1.0), (5000.0, 5.0), (10000.0, 10.0), (20000.0, 20.0),
           (40000.0, 40.0), (50000.0, 50.0), (80000.0, 80.0), (100000.0, 100.0)]             # :151-172, :263-283
_LSE_A = [(0.0, 0.0001), (1.0, 0.0005), (5.0, 0.001), (10.0, 0.005), (50.0, 0.01), (100.0, 0.05),
          (500.0, 0.1), (1000.0, 0.5), (5000.0, 1.0), (10000.0, 5.0)]                        # :216-227
_LSE_B = [(0.0, 0.0001), (0.5, 0.0005), (1.0, 0.001), (5.0, 0.005), (10.0, 0.01), (50.0, 0.05),
          (100.0, 0.1), (500.0, 0.5), (1000.0, 1.0), (5000.0, 5.0), (10000.0, 10.0)]         # :230-242, :294-306 (Swiss)
_LSE_GROUP_A = {"AAL", "BATS", "GSK", "VOD", "HSBA"}
_LSE_GROUP_B = {"BAES", "UU", "LGEN", "LSE", "NXT"}
_MILAN = [(0.0, 0.0001), (0.25, 0.0005), (1.0, 0.001), (2.0, 0.0025), (5.0, 0.005), (50.0, 0.01)]  # :253-261
_VIENNA = [(0.0, 0.001), (10.0, 0.005), (50.0, 0.01), (100.0, 0.5)]                          # :309-313 (0.5 is upstream's)

# venue code -> (table, market open, market close); Market::make_market, market.cpp:40-61
_VENUES = {
    "AS": (_EURONEXT, 9 * HOUR, 17 * HOUR + 40 * MINUTE),   # Amsterdam :176-178
    "BR": (_EURONEXT, 9 * HOUR, 17 * HOUR + 40 * MINUTE),   # Brussels :180-182
    "CO": (_NORDIC, 9 * HOUR, 17 * HOUR),                   # Copenhagen :184-186
    "DE": (_EURONEXT, 9 * HOUR, 17 * HOUR + 30 * MINUTE),   # Xetra :188-192 (same bands as Euronext)
    "HE": (_NORDIC, 10 * HOUR, 16 * HOUR + 30 * MINUTE),    # Helsinki :194-196
    "I": (_EURONEXT, 8 * HOUR, 16 * HOUR + 16 * MINUTE + 40),  # Irish :198-205: add_minutes(16, 40) = 16 min + 40 ms
    "MC": (_EURONEXT, 9 * HOUR, 17 * HOUR + 30 * MINUTE),   # Madrid :247-251
    "MI": (_MILAN, 9 * HOUR, 17 * HOUR + 25 * MINUTE),      # Milan :253-261
    "OL": (_NORDIC, 9 * HOUR, 16 * HOUR + 30 * MINUTE),     # Oslo :263-283
    "PA": (_EURONEXT, 9 * HOUR, 17 * HOUR + 30 * MINUTE),   # Paris :285-287
    "S": (_LSE_B, 9 * HOUR, 17 * HOUR + 30 * MINUTE),       # Swiss :293-307
    "VX": (_LSE_B, 9 * HOUR, 17 * HOUR + 30 * MINUTE),
    "ST": (_NORDIC, 9 * HOUR, 17 * HOUR + 30 * MINUTE),     # Stockholm :289-291
    "VI": (_VIENNA, 9 * HOUR, 17 * HOUR + 30 * MINUTE),     # Vienna :309-313
}


def venue_table(ticker):
    """Market::make_market (src/market/market.cpp:40-61) for 'SYMBOL.VENUE'."""
    symbol, _, venue = ticker.partition(".")
    symbol, venue = symbol.upper(), venue.upper()
    if venue == "L":
        if symbol in _LSE_GROUP_A:
            bands = _LSE_A
        elif symbol in _LSE_GROUP_B:
            bands = _LSE_B
        else:
            raise ValueError('[LondonStockExchange] Unknown symbol "%s".' % symbol)
        return bands, 8 * HOUR, 16 * HOUR + 30 * MINUTE
    if venue in _VENUES:
        return _VENUES[venue]
    raise ValueError('[Market] Unknown exchange venue "%s".' % venue)


def _fill_venue(dst, ticker):
    bands, mo, mc = venue_table(ticker)
    dst.n_bands = len(bands)
    for i, (px, ts) in enumerate(bands):
        dst.band_px[i] = px
        dst.band_ts[i] = ts
    dst.open_ms, dst.close_ms = mo, mc
    return dst


def market(ticker):
    """abi.Market of 'SYMBOL.VENUE' (Market::make_market, src/market/market.cpp:40-61): the tick table and trading hours
    rlm_create takes from the config's first symbol, for rlm_set_day_markets.  Raises as venue_table does."""
    return _fill_venue(abi.Market(), ticker)


def config_market(cfg):
    """abi.Market of a handle's config (its venue block)."""
    m = abi.Market()
    m.n_bands = cfg.n_bands
    for i in range(abi.RLM_MAX_BANDS):
        m.band_px[i] = cfg.band_px[i]
        m.band_ts[i] = cfg.band_ts[i]
    m.open_ms, m.close_ms = cfg.open_ms, cfg.close_ms
    return m


def same_market(a, b):
    """The same tick table and trading hours (unused band slots ignored)."""
    n = a.n_bands
    return (n == b.n_bands and a.open_ms == b.open_ms and a.close_ms == b.close_ms
            and all(a.band_px[i] == b.band_px[i] and a.band_ts[i] == b.band_ts[i] for i in range(n)))


def _get(d, path, default=None, required=False):
    cur = d
    for k in path:
        if not isinstance(cur, dict) or k not in cur:
            if required:
                raise KeyError("missing config key: " + ".".join(path))
            return default
        cur = cur[k]
    return cur


def _f32(x):
    return C.c_float(float(x)).value


def from_dict(y, n_envs=1, ticker=None, device=0, env_index0=0, shared_policy=False,
              source=abi.SOURCE_GENERATOR, algorithm=None, flow_seed=1, dt_ms=250):
    c = abi.Config()
    c.n_envs = n_envs
    c.device = device
    c.env_index0 = env_index0
    c.shared_policy = 1 if shared_policy else 0
    c.source = source
    # learning
    c.memory_size = int(_get(y, ("learning", "memory_size"), required=True))
    c.n_tilings = int(_get(y, ("learning", "n_tilings"), required=True))
    c.n_actions = int(_get(y, ("learning", "n_actions"), required=True))
    algo = algorithm or _get(y, ("learning", "algorithm"), "")
    if algo not in abi.ALGO:
        raise ValueError("Please specify a valid learning algorithm!")  # main.cpp:188-189
    c.algorithm = abi.ALGO[algo]
    c.random_init = 1 if _get(y, ("learning", "random_init"), False) else 0
    gw = _get(y, ("learning", "group_weights"))
    if gw is not None:  # agent.cpp:43-50
        g0, g1 = float(gw[0]), float(gw[1])
        g2 = float(gw[2]) if len(gw) > 2 else 1.0 - (g0 + g1)
    else:
        g0 = g1 = g2 = 1.0 / 3
    c.group_weights[0], c.group_weights[1], c.group_weights[2] = g0, g1, g2
    c.gamma = float(_get(y, ("learning", "gamma"), required=True))
    c.lambda_ = float(_get(y, ("learning", "lambda"), required=True))
    c.omega = float(_get(y, ("learning", "omega"), 1.0))
    c.alpha_start = float(_get(y, ("learning", "alpha_start"), 0.2))
    c.alpha_floor = float(_get(y, ("learning", "alpha_floor"), 0.001))
    c.beta = float(_get(y, ("learning", "beta"), 0.0))
    # policy
    pt = _get(y, ("policy", "type"), "")
    if pt not in abi.POLICY:
        raise ValueError("Please specify a valid policy!")  # main.cpp:164-165
    c.policy_type = abi.POLICY[pt]
    c.eps_init = _f32(_get(y, ("policy", "eps_init"), 0.0))
    c.eps_floor = _f32(_get(y, ("policy", "eps_floor"), 0.0))
    c.eps_T = int(_get(y, ("policy", "eps_T"), 1))
    c.tau_init = _f32(_get(y, ("policy", "tau_init"), 1.0))
    c.tau_floor = _f32(_get(y, ("policy", "tau_floor"), 1.0))
    c.tau_T = int(_get(y, ("policy", "tau_T"), 1))
    c.spread_lookback = int(_get(y, ("policy", "spread_lookback"), 10))
    # reward
    rm = _get(y, ("reward", "measure"), "pnl")
    if rm not in abi.REWARD:
        raise ValueError("Unknown reward measure: " + str(rm))  # base.cpp:74-75
    c.reward_measure = abi.REWARD[rm]
    c.damping_factor = _f32(_get(y, ("reward", "damping_factor"), 1.0))
    c.pos_weight = _f32(_get(y, ("reward", "pos_weight"), 0.0))
    c.trd_weight = _f32(_get(y, ("reward", "trd_weight"), 0.0))
    c.pnl_weight = _f32(_get(y, ("reward", "pnl_weight"), 1.0))
    c.pnl_lookback = int(_get(y, ("reward", "pnl_lookback"), 0))
    # state
    sv = _get(y, ("state", "variables"), required=True)
    if len(sv) > abi.RLM_N_STATE_MAX:
        raise ValueError("too many state variables")
    c.n_state_vars = len(sv)
    for i, name in enumerate(sv):
        if name not in abi.VAR:
            raise ValueError("Unknown state variable: %s." % name)  # intraday.cpp:57-60
        c.state_vars[i] = abi.VAR[name]
    c.lb_mpm = int(_get(y, ("state", "lookback", "mpm"), 0))
    c.lb_vlt = int(_get(y, ("state", "lookback", "vlt"), 0))
    c.lb_svl = int(_get(y, ("state", "lookback", "svl"), 0))
    c.lb_rsi = int(_get(y, ("state", "lookback", "rsi"), 0))
    c.lb_vwap = int(_get(y, ("state", "lookback", "vwap"), 0))
    # market
    c.pos_lb = int(_get(y, ("market", "pos_lb"), required=True))
    c.pos_ub = int(_get(y, ("market", "pos_ub"), required=True))
    c.order_size = int(_get(y, ("market", "order_size"), 1))
    tp = _get(y, ("market", "target_price", "type"), "midprice")
    c.target_price_type = abi.TP_YAML.get(tp, abi.TP_YAML["microprice"])  # any other string -> tp::MidPrice
    c.tp_lookback = int(_get(y, ("market", "target_price", "lookback"), 1))
    lat = _get(y, ("market", "latency", "type"), "fixed")
    if lat not in ("fixed", "normal", "lognormal"):
        raise ValueError("Unknown latency type: " + str(lat))  # base.cpp:94-95
    # The sampler itself is not built: its only consumer writes Intraday::ref_time (intraday.cpp:178), which nothing reads,
    # and it draws from a generator of its own (latency.cpp:19-22) -- no observable effect.  Its constructor checks are kept.
    if float(_get(y, ("market", "latency", "floor"), 0.0)) < 0.0:
        raise ValueError("Latency must be zero or positive.")  # latency.cpp:12-13
    if lat == "normal" and _get(y, ("market", "latency", "sigma"), None) is None:
        raise ValueError("market.latency.sigma is required for the normal latency (base.cpp:86)")
    if lat == "lognormal" and _get(y, ("market", "latency", "beta"), None) is None:
        raise ValueError("market.latency.beta is required for the lognormal latency (base.cpp:91)")
    # venue
    if ticker is None:
        syms = _get(y, ("data", "symbols"), ["AAL.L"])
        ticker = syms[0]
    _fill_venue(c, ticker)
    # debug
    seed = _get(y, ("debug", "random_seed"))
    if seed is None:
        raise ValueError("debug.random_seed must be set: the reference falls back to the wall clock "
                         "(main.cpp:84-85), which is not reproducible")
    c.random_seed = int(seed)
    set_default_flow(c, flow_seed, dt_ms)
    return c


def set_default_flow(c, seed, dt_ms):
    """rlm_flow_default_params (include/rlm_flow.h)."""
    f = c.flow
    f.seed = seed
    f.mid0_tick = 52500
    f.tick_lo = 49000 + 400
    f.tick_hi = 57000 - 400
    f.band_tick0 = 49000
    f.dt_ms = dt_ms
    # first row right after the venue's open + 30 min guard (market.cpp:67-70); LSE: 08:30:00.000 as in rlm_flow.h
    f.t0_ms = int(c.open_ms) + 30 * MINUTE if c.open_ms else 8 * HOUR + 30 * MINUTE
    f.date = 20100104
    f.vol0 = 500
    f.p_move_u12 = 1024
    f.p_spread_u12 = 410
    f.spread_c1_u12 = 2048
    f.spread_c2_u12 = 3277
    f.p_deep_u2 = 1
    f.band_px0 = 1000.0
    f.band_ts = 0.5


def from_yaml(path, **kw):
    with open(path) as fh:
        return from_dict(yaml.safe_load(fh), **kw)


EXAMPLE_YAML = """
debug:
    inspect_books: false
    random_seed: 1994
training:
    n_threads: 1
    n_samples: 1
    n_episodes: 1000
evaluation:
    n_samples: 20
    use_train_sample: false
    random_agent: false
learning:
    memory_size: 65536
    n_tilings: 32
    n_actions: 9
    algorithm: q_learn
    group_weights: [0.65, 0.25, 0.10]
    gamma: 0.975
    lambda: 0.85
    omega: 1.0
    alpha_start: 0.001
    alpha_floor: 0.001
    beta: 0.005
policy:
    type: epsilon_greedy
    eps_init: 0.8
    eps_floor: 0.0001
    eps_T: 800
    spread_lookback: 45
reward:
    measure: pnl_damped
    damping_factor: 0.15
    pnl_lookback: 0
    pos_weight: 0.0
    pnl_weight: 1.0
state:
    variables: ["pos", "a_dist", "b_dist", "mpm", "spd", "vol", "imb", "svl"]
    lookback:
        mpm: 15
        vlt: 60
        svl: 60
        rsi: 0
        vwap: 0
data:
    symbols: ["AAL.L"]
market:
    transaction_fee: 0.0
    target_price:
        type: midprice
        lookback: 1
    latency:
        type: fixed
        floor: 0.0
        mu: 0.0
        sigma: 0.0
    pos_ub: 50
    pos_lb: -50
    order_size: 10
"""


def example_dict(**overrides):
    """config/example.yaml with the parity-run settings of SURVEY.md section 8d (C0): explicit seed,
    symbol AAL.L, q_learn, per-env memory_size.  `overrides` uses dotted keys: learning.memory_size=4096."""
    y = yaml.safe_load(EXAMPLE_YAML)
    for k, v in overrides.items():
        cur = y
        parts = k.split(".")
        for p in parts[:-1]:
            cur = cur.setdefault(p, {})
        cur[parts[-1]] = v
    return y
