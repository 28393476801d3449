"""ctypes mirror of include/rlm.h, include/rlm_flow.h and include/rlm_record.h.

Plain-C structures only; nothing here touches torch.  These are the structures of the
product library (rl_markets_b200/csrc -> librlm.so); the test-side checker speaks the same
C structs but is never imported from here.
"""
import ctypes as C

RLM_DEPTH = 5
RLM_N_TX_MAX = 4
RLM_N_STATE_MAX = 13
RLM_MAX_BANDS = 32
RLM_MAX_ACTIONS = 9
RLM_N_TILINGS = 32
RLM_EVAL_Q_CHUNK = 1 << 17  # queries per device pass of rlm_eval_q
# checkpoint files (rlm_save): the model_log capacity and the saved rlm_config sit at fixed offsets of the header
CKPT_MODEL_LOG_CAP_OFFSET = 40
CKPT_CONFIG_OFFSET = 48

# enums (include/rlm.h)
ALGO = {"q_learn": 0, "sarsa": 1, "double_q_learn": 2, "r_learn": 3, "online_r_learn": 4, "double_r_learn": 5}
POLICY = {"greedy": 0, "random": 1, "epsilon_greedy": 2, "boltzmann": 3}
REWARD = {"none": 0, "pnl": 1, "pnl_damped": 2, "spread": 3, "normed": 4, "lovol": 5, "mm_linear": 6,
          "mm_exp": 7, "mm_div": 8}
VAR = {"pos": 0, "spd": 1, "mpm": 2, "imb": 3, "svl": 4, "vol": 5, "rsi": 6, "vwap": 7, "a_dist": 8,
       "a_queue": 9, "b_dist": 10, "b_queue": 11, "last_action": 12}
TP_YAML = {"midprice": 0, "microprice": 1, "vwap": 2, "book": 3}
MODE_TRAIN, MODE_BACKTEST = 0, 1
SOURCE_GENERATOR, SOURCE_STREAM, SOURCE_TAPE = 0, 1, 2
TICK_PARTIAL, TICK_TX_MORE = 1, 2  # rlm_tick_msg.flags (include/rlm_flow.h)

RLM_OK = 0
RLM_ERR_INVALID_ARGUMENT = -1
RLM_ERR_RUNTIME = -2
RLM_ERR_NO_DEVICE = -3
RLM_ERR_CUDA = -4
RLM_ERR_UNSUPPORTED = -5
RLM_ERR_END_OF_DATA = -6


class TickMsg(C.Structure):
    _fields_ = [
        ("ask_px", C.c_float * RLM_DEPTH),
        ("bid_px", C.c_float * RLM_DEPTH),
        ("ask_vol", C.c_int32 * RLM_DEPTH),
        ("bid_vol", C.c_int32 * RLM_DEPTH),
        ("tx_px", C.c_float * RLM_N_TX_MAX),
        ("tx_vol", C.c_int32 * RLM_N_TX_MAX),
        ("n_tx", C.c_int32),
        ("time_ms", C.c_int32),
        ("date", C.c_int32),
        ("flags", C.c_int32),
    ]


assert C.sizeof(TickMsg) == 128


class FlowParams(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64),
        ("mid0_tick", C.c_int32),
        ("tick_lo", C.c_int32),
        ("tick_hi", C.c_int32),
        ("band_tick0", C.c_int32),
        ("dt_ms", C.c_int32),
        ("t0_ms", C.c_int32),
        ("date", C.c_int32),
        ("vol0", C.c_int32),
        ("p_move_u12", C.c_int32),
        ("p_spread_u12", C.c_int32),
        ("spread_c1_u12", C.c_int32),
        ("spread_c2_u12", C.c_int32),
        ("p_deep_u2", C.c_int32),
        ("band_px0", C.c_float),
        ("band_ts", C.c_float),
    ]


class OrderRec(C.Structure):
    _fields_ = [
        ("exists", C.c_int32),
        ("pad", C.c_int32),
        ("price", C.c_double),
        ("q_head", C.c_int64),
        ("q_tail", C.c_int64),
        ("executed", C.c_int64),
    ]


class StepRecord(C.Structure):
    _fields_ = [
        ("step", C.c_int32),
        ("action", C.c_int32),
        ("time_ms", C.c_int32),
        ("terminal", C.c_int32),
        ("position", C.c_int64),
        ("ask_quote", C.c_double),
        ("bid_quote", C.c_double),
        ("ask_level", C.c_int32),
        ("bid_level", C.c_int32),
        ("reward", C.c_double),
        ("pnl_step", C.c_double),
        ("ep_pnl", C.c_double),
        ("ep_reward", C.c_double),
        ("ep_bandh", C.c_double),
        ("midprice", C.c_double),
        ("spread", C.c_double),
        ("bandh_step", C.c_double),
        ("ask", OrderRec),
        ("bid", OrderRec),
        ("ask_transactions", C.c_int32),
        ("bid_transactions", C.c_int32),
        ("market_buys", C.c_int32),
        ("market_sells", C.c_int32),
        ("lo_vol_step", C.c_int32),
        ("n_state", C.c_int32),
        ("state", C.c_float * (RLM_N_STATE_MAX + 1)),
        ("delta", C.c_double),
        ("n_traces", C.c_int32),
        ("pad", C.c_int32),
        ("trace_hash", C.c_uint64),
    ]


class Config(C.Structure):
    _fields_ = [
        ("n_envs", C.c_int32),
        ("device", C.c_int32),
        ("env_index0", C.c_int64),
        ("shared_policy", C.c_int32),
        ("source", C.c_int32),
        ("memory_size", C.c_int64),
        ("n_tilings", C.c_int32),
        ("n_actions", C.c_int32),
        ("algorithm", C.c_int32),
        ("random_init", C.c_int32),
        ("group_weights", C.c_double * 3),
        ("gamma", C.c_double),
        ("lambda_", C.c_double),
        ("omega", C.c_double),
        ("alpha_start", C.c_double),
        ("alpha_floor", C.c_double),
        ("beta", C.c_double),
        ("policy_type", C.c_int32),
        ("eps_init", C.c_float),
        ("eps_floor", C.c_float),
        ("eps_T", C.c_uint32),
        ("tau_init", C.c_float),
        ("tau_floor", C.c_float),
        ("tau_T", C.c_uint32),
        ("spread_lookback", C.c_int32),
        ("reward_measure", C.c_int32),
        ("damping_factor", C.c_float),
        ("pos_weight", C.c_float),
        ("trd_weight", C.c_float),
        ("pnl_weight", C.c_float),
        ("pnl_lookback", C.c_int32),
        ("n_state_vars", C.c_int32),
        ("state_vars", C.c_int32 * RLM_N_STATE_MAX),
        ("lb_mpm", C.c_int32),
        ("lb_vlt", C.c_int32),
        ("lb_svl", C.c_int32),
        ("lb_rsi", C.c_int32),
        ("lb_vwap", C.c_int32),
        ("pos_lb", C.c_int64),
        ("pos_ub", C.c_int64),
        ("order_size", C.c_int32),
        ("target_price_type", C.c_int32),
        ("tp_lookback", C.c_int32),
        ("n_bands", C.c_int32),
        ("band_px", C.c_double * RLM_MAX_BANDS),
        ("band_ts", C.c_double * RLM_MAX_BANDS),
        ("open_ms", C.c_int64),
        ("close_ms", C.c_int64),
        ("random_seed", C.c_uint32),
        ("flow", FlowParams),
        ("trace_cap", C.c_int32),
        ("record_envs", C.c_int32),
        ("record_cap", C.c_int32),
        ("reserved", C.c_int32 * 5),
    ]


class Market(C.Structure):
    """rlm_market: one venue's tick table and trading hours (rlm_set_day_markets)."""
    _fields_ = [
        ("n_bands", C.c_int32),
        ("pad", C.c_int32),
        ("band_px", C.c_double * RLM_MAX_BANDS),
        ("band_ts", C.c_double * RLM_MAX_BANDS),
        ("open_ms", C.c_int64),
        ("close_ms", C.c_int64),
    ]


class Counters(C.Structure):
    _fields_ = [
        ("ticks", C.c_int64),
        ("steps", C.c_int64),
        ("sum_traces", C.c_int64),
        ("terminal_envs", C.c_int64),
        ("kernel_launches", C.c_int64),
    ]


class EnvStats(C.Structure):
    _fields_ = [
        ("episode_reward", C.c_double),
        ("episode_pnl", C.c_double),
        ("episode_bandh", C.c_double),
        ("position", C.c_int64),
        ("ask_transactions", C.c_int32),
        ("bid_transactions", C.c_int32),
        ("market_buys", C.c_int32),
        ("market_sells", C.c_int32),
        ("total_ticks", C.c_int32),
        ("steps", C.c_int32),
        ("terminal", C.c_int32),
        ("phase", C.c_int32),
    ]


class OrderOp(C.Structure):
    _fields_ = [("op", C.c_int32), ("pad", C.c_int32), ("arg", C.c_int64)]


class OrderState(C.Structure):
    _fields_ = [("size", C.c_int64), ("q_head", C.c_int64), ("q_tail", C.c_int64), ("executed", C.c_int64),
                ("ret", C.c_int64)]


def record_fields_equal(a, b, skip=()):
    """Bitwise comparison of two StepRecord instances; returns list of differing field names."""
    bad = []
    for name, typ in StepRecord._fields_:
        if name in skip or name == "pad":
            continue
        va, vb = getattr(a, name), getattr(b, name)
        if isinstance(va, C.Array):
            if bytes(va) != bytes(vb):
                bad.append(name)
        elif isinstance(va, C.Structure):
            if bytes(va) != bytes(vb):
                bad.append(name)
        elif typ is C.c_double:
            if C.c_double(va).value != C.c_double(vb).value and not (va != va and vb != vb):
                bad.append(name)
            elif bytes(C.c_double(va)) != bytes(C.c_double(vb)):
                bad.append(name)
        elif va != vb:
            bad.append(name)
    return bad
