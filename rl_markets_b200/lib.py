"""ctypes binding of librlm.so (the C ABI of include/rlm.h).

The library is built in-tree by rl_markets_b200/csrc/Makefile (see __graft_entry__.build).
There is no CPU fallback: if the extension is missing, or no CUDA device is usable,
every entry point raises.
"""
import ctypes as C
import os

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RLM_LIB_PATH") or os.path.join(_HERE, "librlm.so")  # (RLM_LIB_PATH: the phase-timeline build of tools/phase_probe.py)

EXPORTS = [
    "rlm_last_error", "rlm_abi_version", "rlm_config_default", "rlm_create", "rlm_destroy", "rlm_reset", "rlm_set_mode", "rlm_new_env", "rlm_set_flow",
    "rlm_load_ticks", "rlm_load_days", "rlm_assign_days", "rlm_get_tape_pos", "rlm_set_day_markets", "rlm_run_ticks", "rlm_sync", "rlm_get_counters", "rlm_get_stats", "rlm_get_state",
    "rlm_get_reward", "rlm_get_actions", "rlm_get_rho", "rlm_get_occupancy", "rlm_copy_theta", "rlm_handle_terminal", "rlm_go_greedy", "rlm_read_theta",
    "rlm_write_theta", "rlm_save", "rlm_load", "rlm_eval_q", "rlm_set_model_log", "rlm_read_model_log", "rlm_get_policy_descr", "rlm_read_records", "rlm_device_ptrs", "rlm_shared_tick_accumulate", "rlm_apply_dtheta",
    "rlm_set_stream", "rlm_set_profiling", "rlm_get_kernel_times", "rlm_act", "rlm_env_step", "rlm_agent_update", "rlm_ingest_csv",
    "rlm_flow_generate", "rlm_test_to_ticks", "rlm_test_to_price", "rlm_test_tiles", "rlm_test_learner_tiles", "rlm_test_order",
    "rlm_test_rolling_mean",
]


class RlmError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("rlm status %d: %s" % (code, msg))
        self.code = code


_lib = None


def load():
    """Load librlm.so; raises (never falls back to anything else) if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RlmError(abi.RLM_ERR_NO_DEVICE,
                       "librlm.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                       "there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.rlm_last_error.restype = C.c_char_p
    P = C.POINTER
    L.rlm_config_default.argtypes = [P(abi.Config)]
    L.rlm_create.argtypes = [P(abi.Config), P(C.c_void_p)]
    L.rlm_destroy.argtypes = [C.c_void_p]
    L.rlm_reset.argtypes = [C.c_void_p]
    L.rlm_set_mode.argtypes = [C.c_void_p, C.c_int32]
    L.rlm_new_env.argtypes = [C.c_void_p, P(abi.FlowParams)]
    L.rlm_set_flow.argtypes = [C.c_void_p, P(abi.FlowParams)]
    L.rlm_load_ticks.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.rlm_load_days.argtypes = [C.c_void_p, C.c_void_p, P(C.c_int64), C.c_int32]
    L.rlm_assign_days.argtypes = [C.c_void_p, C.c_int32, C.c_int32, P(C.c_int32)]
    L.rlm_get_tape_pos.argtypes = [C.c_void_p, P(C.c_int64)]
    L.rlm_set_day_markets.argtypes = [C.c_void_p, P(abi.Market), C.c_int32, P(C.c_int32), C.c_int32]
    L.rlm_run_ticks.argtypes = [C.c_void_p, C.c_int32]
    L.rlm_sync.argtypes = [C.c_void_p]
    L.rlm_get_counters.argtypes = [C.c_void_p, P(abi.Counters)]
    L.rlm_get_stats.argtypes = [C.c_void_p, C.c_int32, C.c_int32, P(abi.EnvStats)]
    L.rlm_get_state.argtypes = [C.c_void_p, P(C.c_float)]
    L.rlm_get_reward.argtypes = [C.c_void_p, P(C.c_double)]
    L.rlm_get_actions.argtypes = [C.c_void_p, P(C.c_int32)]
    L.rlm_get_rho.argtypes = [C.c_void_p, P(C.c_double)]
    L.rlm_get_occupancy.argtypes = [C.c_void_p, P(C.c_int32)]
    L.rlm_copy_theta.argtypes = [C.c_void_p, C.c_void_p]
    L.rlm_handle_terminal.argtypes = [C.c_void_p, C.c_int32]
    L.rlm_go_greedy.argtypes = [C.c_void_p]
    L.rlm_read_theta.argtypes = [C.c_void_p, C.c_int32, C.c_int32, P(C.c_double), C.c_int64]
    L.rlm_write_theta.argtypes = [C.c_void_p, C.c_int32, C.c_int32, P(C.c_double), C.c_int64]
    L.rlm_save.argtypes = [C.c_void_p, C.c_char_p]
    L.rlm_load.argtypes = [C.c_void_p, C.c_char_p]
    L.rlm_eval_q.argtypes = [C.c_void_p, P(C.c_float), P(C.c_int32), C.c_int64, P(C.c_double)]
    L.rlm_set_model_log.argtypes = [C.c_void_p, C.c_int64]
    L.rlm_read_model_log.argtypes = [C.c_void_p, C.c_int32, C.c_int32, P(C.c_double), P(C.c_int32)]
    L.rlm_get_policy_descr.argtypes = [C.c_void_p, P(C.c_double)]
    L.rlm_read_records.argtypes = [C.c_void_p, C.c_int32, P(abi.StepRecord), C.c_int32, P(C.c_int32)]
    L.rlm_device_ptrs.argtypes = [C.c_void_p, P(C.c_void_p), P(C.c_void_p), P(C.c_int64)]
    L.rlm_apply_dtheta.argtypes = [C.c_void_p]
    L.rlm_shared_tick_accumulate.argtypes = [C.c_void_p]
    L.rlm_act.argtypes = [C.c_void_p, P(C.c_int32)]
    L.rlm_env_step.argtypes = [C.c_void_p, P(C.c_int32), P(C.c_double), P(C.c_uint8)]
    L.rlm_agent_update.argtypes = [C.c_void_p, P(C.c_double)]
    L.rlm_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    L.rlm_set_profiling.argtypes = [C.c_void_p, C.c_int32]
    L.rlm_get_kernel_times.argtypes = [C.c_void_p, P(C.c_double), P(C.c_double), P(C.c_int64), P(C.c_int64)]
    L.rlm_ingest_csv.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int64, P(C.c_int64), P(C.c_int64)]
    L.rlm_flow_generate.argtypes = [P(abi.FlowParams), C.c_int64, C.c_int64, C.c_int32, P(abi.TickMsg)]
    L.rlm_test_to_ticks.argtypes = [P(abi.Config), P(C.c_double), C.c_int32, P(C.c_int32)]
    L.rlm_test_to_price.argtypes = [P(abi.Config), P(C.c_int32), C.c_int32, P(C.c_double)]
    L.rlm_test_tiles.argtypes = [P(abi.Config), P(C.c_float), C.c_int32, P(C.c_int32)]
    L.rlm_test_learner_tiles.argtypes = [P(abi.Config), C.c_int32, P(C.c_float), C.c_int32, P(C.c_int32)]
    L.rlm_test_order.argtypes = [C.c_int64, C.c_int64, P(abi.OrderOp), C.c_int32, P(abi.OrderState)]
    L.rlm_test_rolling_mean.argtypes = [C.c_int32, P(C.c_double), C.c_int32, P(C.c_double)]
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise RlmError(rc, load().rlm_last_error().decode())


def flow_generate(flow_params, env_index, first_tick, n_ticks):
    """Host rendering of the synthetic flow (same integer process as the in-kernel generator)."""
    out = (abi.TickMsg * n_ticks)()
    check(load().rlm_flow_generate(C.byref(flow_params), env_index, first_tick, n_ticks, out))
    return out


def ingest_csv(md_path, tas_path):
    """Reference-format CSV pair -> (ctypes array of TickMsg, number of market ticks); see rlm_ingest_csv in include/rlm.h."""
    L = load()
    n, t = C.c_int64(0), C.c_int64(0)
    check(L.rlm_ingest_csv(md_path.encode(), tas_path.encode(), None, 0, C.byref(n), C.byref(t)))
    out = (abi.TickMsg * max(n.value, 1))()
    check(L.rlm_ingest_csv(md_path.encode(), tas_path.encode(), C.addressof(out), n.value, C.byref(n), C.byref(t)))
    return out, n.value, t.value


class BatchedMarket:
    """B independent (Intraday env + agent + learner) triples on one GPU.

    Mirrors the call order of experiment::serial::Learner::RunEpisode
    (src/experiment/serial.cpp:72-94): construct -> [load_ticks] -> run_ticks ... ->
    handle_terminal(episode) -> reset.
    """

    def __init__(self, cfg):
        self.L = load()
        self.cfg = cfg
        self.h = C.c_void_p()
        check(self.L.rlm_create(C.byref(cfg), C.byref(self.h)))
        self._keep = None

    def close(self):
        if self.h:
            self.L.rlm_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        check(self.L.rlm_reset(self.h))

    def set_mode(self, mode):
        """abi.MODE_TRAIN (Learner::_step) or abi.MODE_BACKTEST (Backtester::_step, serial.cpp:121-137)."""
        check(self.L.rlm_set_mode(self.h, mode))

    def new_env(self, flow=None):
        """Fresh env objects for the same agents (main.cpp:219); `flow` = synthetic-flow parameters of the new day."""
        check(self.L.rlm_new_env(self.h, C.byref(flow) if flow is not None else None))
        if flow is not None:
            self.cfg.flow = flow

    def set_flow(self, flow):
        """LoadData of another synthetic day on the same env objects (generator source); follow with reset().  The
        next test day of main.cpp:219-241, whose env object outlives the day (new_env is the first test day only)."""
        check(self.L.rlm_set_flow(self.h, C.byref(flow)))
        self.cfg.flow = flow

    def load_ticks(self, msgs, n_ticks):
        """msgs: ctypes array (or address) of TickMsg laid out [tick][env]; kept alive until sync()."""
        self._keep = msgs
        addr = msgs if isinstance(msgs, int) else C.addressof(msgs)
        check(self.L.rlm_load_ticks(self.h, addr, n_ticks))

    def load_days(self, msgs, offsets):
        """Tape source: upload a library of days once (rlm_load_days).  msgs: ctypes array (or address) of TickMsg, the days
        one after the other; offsets: n_days + 1 message offsets (day d = msgs[offsets[d]:offsets[d + 1]]).  Env b replays
        day b % n_days from its start."""
        offs = (C.c_int64 * len(offsets))(*offsets)
        addr = msgs if isinstance(msgs, int) else C.addressof(msgs)
        check(self.L.rlm_load_days(self.h, addr, offs, len(offsets) - 1))

    def assign_days(self, days, env0=0):
        """Tape source: env env0 + i replays day days[i] from its first message (Intraday::LoadData per env)."""
        n = len(days)
        check(self.L.rlm_assign_days(self.h, env0, n, (C.c_int32 * max(n, 1))(*days)))

    def set_day_markets(self, markets, day_market):
        """Tape source: day d runs under markets[day_market[d]] (abi.Market, e.g. config.market(ticker)); rewinds every env
        to the start of its day, follow with reset().  A later load_days drops them (rlm_set_day_markets)."""
        arr = (abi.Market * max(len(markets), 1))(*markets)
        dm = (C.c_int32 * max(len(day_market), 1))(*day_market)
        check(self.L.rlm_set_day_markets(self.h, arr, len(markets), dm, len(day_market)))

    def load_day_library(self, samples):
        """Tape source: the (symbol, md csv, tas csv) days of ingest.file_sample / sample_window into this handle, each
        under its symbol's market.  Day markets are set only when some day's market differs from the config's, so a
        library of one market keeps the kernels without day markets.  Returns the number of days."""
        from . import config, ingest
        msgs, offsets = ingest.day_library(samples)
        self.load_days(msgs, offsets)
        markets, day_market = ingest.day_markets(samples)
        mine = config.config_market(self.cfg)
        if not all(config.same_market(m, mine) for m in markets):
            self.set_day_markets(markets, day_market)
        return len(samples)

    def tape_pos(self):
        """Tape source: messages of its day each env has consumed since it was assigned or rewound."""
        out = (C.c_int64 * self.cfg.n_envs)()
        check(self.L.rlm_get_tape_pos(self.h, out))
        return list(out)

    def run_ticks(self, n):
        check(self.L.rlm_run_ticks(self.h, n))

    def sync(self):
        check(self.L.rlm_sync(self.h))

    def set_stream(self, cuda_stream_ptr):
        check(self.L.rlm_set_stream(self.h, cuda_stream_ptr))
        self._stream_ptr = cuda_stream_ptr

    def counters(self):
        c = abi.Counters()
        check(self.L.rlm_get_counters(self.h, C.byref(c)))
        return c

    def stats(self, env0=0, n=None):
        n = self.cfg.n_envs - env0 if n is None else n
        out = (abi.EnvStats * n)()
        check(self.L.rlm_get_stats(self.h, env0, n, out))
        return out

    def state(self):
        out = (C.c_float * (self.cfg.n_envs * self.cfg.n_state_vars))()
        check(self.L.rlm_get_state(self.h, out))
        return out

    def rewards(self):
        out = (C.c_double * self.cfg.n_envs)()
        check(self.L.rlm_get_reward(self.h, out))
        return out

    def actions(self):
        out = (C.c_int32 * self.cfg.n_envs)()
        check(self.L.rlm_get_actions(self.h, out))
        return out

    def rho(self):
        out = (C.c_double * self.cfg.n_envs)()
        check(self.L.rlm_get_rho(self.h, out))
        return out

    def copy_theta_from(self, other):
        """Take over the trained weights of another handle (same shape, same device)."""
        check(self.L.rlm_copy_theta(self.h, other.h))

    def occupancy(self):
        """Written weights per env (population of the gather-skipping bitmap); diagnostic."""
        out = (C.c_int32 * self.cfg.n_envs)()
        check(self.L.rlm_get_occupancy(self.h, out))
        return out

    def handle_terminal(self, episode):
        check(self.L.rlm_handle_terminal(self.h, episode))

    def go_greedy(self):
        check(self.L.rlm_go_greedy(self.h))

    def theta(self, policy=0, table=0):
        n = self.cfg.memory_size
        out = (C.c_double * n)()
        check(self.L.rlm_read_theta(self.h, policy, table, out, n))
        return out

    def write_theta(self, values, policy=0, table=0):
        """Load one weight table (memory_size doubles; table 1 = Q_B of the double agents) into policy `policy` -- policy 0 is
        the only one of a shared_policy handle: load a trained policy there, go_greedy(), set_mode(MODE_BACKTEST) and every
        env evaluates it on its own day."""
        n = self.cfg.memory_size
        buf = values if isinstance(values, C.Array) and values._type_ is C.c_double else (C.c_double * n).from_buffer_copy(bytes(values))
        assert len(buf) == n, (len(buf), n)
        check(self.L.rlm_write_theta(self.h, policy, table, buf, n))

    # ---- checkpoints (rlm_save / rlm_load)
    def save(self, path):
        """Write every piece of this handle's state to one file (rlm_save); load() into a handle of the same config resumes
        the run bit for bit."""
        check(self.L.rlm_save(self.h, os.fsencode(path)))

    def load(self, path):
        """Resume the handle saved in `path` (rlm_load).  The handle must have been created with the same config (device and
        flow aside) and, on the tape source, hold the same day library.  Takes over the file's flow parameters and model_log
        capacity."""
        check(self.L.rlm_load(self.h, os.fsencode(path)))
        with open(path, "rb") as f:
            head = f.read(abi.CKPT_CONFIG_OFFSET + C.sizeof(abi.Config))
        self._mlog_cap = int.from_bytes(head[abi.CKPT_MODEL_LOG_CAP_OFFSET:abi.CKPT_MODEL_LOG_CAP_OFFSET + 8], "little", signed=True)
        self.cfg.flow = abi.Config.from_buffer_copy(head, abi.CKPT_CONFIG_OFFSET).flow

    @property
    def n_tables(self):
        return 2 if self.cfg.algorithm in (abi.ALGO["double_q_learn"], abi.ALGO["double_r_learn"]) else 1

    def q_values(self, vars=None, policy=None):
        """Agent::getQ / DoubleAgent::getQb (rlm_eval_q) -> float64 array [n][n_tables][n_actions]; [:, 1] is Q_B.

        vars: float32 array [n][n_state_vars], tile-coded as State::newState(vars, .) does, each row under the theta of
        policy[i] (int32 [n]; None = policy 0).  vars=None: the live form, Q of every env's current decision state under its
        own policy (the values Agent::action samples from between agent_update and act).  The call only reads theta."""
        import numpy as np
        T, A, nv = self.n_tables, self.cfg.n_actions, self.cfg.n_state_vars
        if vars is None:
            if policy is not None:
                raise ValueError("q_values: the live form (vars=None) evaluates each env under its own policy; policy must be None")
            n, vp = self.cfg.n_envs, None
        else:
            vars = np.asarray(vars)
            if vars.dtype != np.float32:
                raise TypeError("q_values: vars must be float32, got %s" % vars.dtype)
            if vars.ndim != 2 or vars.shape[1] != nv:
                raise ValueError("q_values: vars must have shape (n, %d), got %s" % (nv, vars.shape))
            vars = np.ascontiguousarray(vars)
            n, vp = vars.shape[0], vars.ctypes.data_as(C.POINTER(C.c_float))
        pp = None
        if policy is not None:
            policy = np.asarray(policy)
            if policy.dtype != np.int32:
                raise TypeError("q_values: policy must be int32, got %s" % policy.dtype)
            if policy.shape != (n,):
                raise ValueError("q_values: policy must have shape (%d,), got %s" % (n, policy.shape))
            policy = np.ascontiguousarray(policy)
            pp = policy.ctypes.data_as(C.POINTER(C.c_int32))
        out = np.empty((n, T, A), dtype=np.float64)
        check(self.L.rlm_eval_q(self.h, vp, pp, n, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    # ---- training logs (logging.log_learning; rl_markets_b200/train_logs.py writes the files)
    def set_model_log(self, cap_rows):
        """Agent::HandleTransition's model_log on the device: cap_rows > 0 keeps up to cap_rows logged values per env between
        two model_log() reads, starting from the Agent constructor's state; 0 turns it off (rlm_set_model_log)."""
        if not isinstance(cap_rows, int) or isinstance(cap_rows, bool):
            raise TypeError("set_model_log: cap_rows must be an int, got %r" % (cap_rows,))
        check(self.L.rlm_set_model_log(self.h, cap_rows))
        self._mlog_cap = cap_rows

    def model_log(self, env0=0, n=None):
        """Drain the model_log of envs env0 .. env0+n-1: one list of floats per env (_agg_delta / 1000 of every 1000th
        update since the last read, in order).  Raises RlmError when an env logged more than cap_rows values in between."""
        n = self.cfg.n_envs - env0 if n is None else n
        cap = getattr(self, "_mlog_cap", 0)
        rows = (C.c_double * max(n * cap, 1))()
        cnt = (C.c_int32 * max(n, 1))()
        check(self.L.rlm_read_model_log(self.h, env0, n, rows, cnt))
        return [[rows[i * cap + k] for k in range(cnt[i])] for i in range(n)]

    def policy_descr(self):
        """Policy::descr(): eps / tau after the last handle_terminal, 0 for greedy and random policies (training_log's last
        column)."""
        out = C.c_double()
        check(self.L.rlm_get_policy_descr(self.h, C.byref(out)))
        return out.value

    def set_profiling(self, on):
        check(self.L.rlm_set_profiling(self.h, 1 if on else 0))

    def kernel_times(self):
        a, b, na, nb = C.c_double(), C.c_double(), C.c_int64(), C.c_int64()
        check(self.L.rlm_get_kernel_times(self.h, C.byref(a), C.byref(b), C.byref(na), C.byref(nb)))
        return {"env_ms": a.value, "agent_ms": b.value, "env_launches": na.value, "agent_launches": nb.value}

    # ---- split surface: Environment::step / Agent::update (include/rlm.h).  Train mode: Learner::_step (independent
    # policies); backtest mode: Backtester::_step (independent and shared policies)
    def act(self):
        """Agent::action for every env at a decision point (-1 elsewhere, and where the episode is over).  Backtest mode:
        the greedy action from the state the last agent_update built."""
        out = (C.c_int32 * self.cfg.n_envs)()
        check(self.L.rlm_act(self.h, out))
        return out

    def env_step(self, actions=None):
        """Base::performAction + getReward: one learner step's worth of ticks per env.  Returns (rewards, terminal):
        terminal[b] is 1 when env b's episode is over, 2 when its tape day ran out inside performAction (tape source).
        actions given without act(): the caller's own actions (no policy draw), in either mode."""
        n = self.cfg.n_envs
        rew, term = (C.c_double * n)(), (C.c_uint8 * n)()
        check(self.L.rlm_env_step(self.h, actions, rew, term))
        return rew, term

    def agent_update(self):
        """Train mode: State::newState + Agent::HandleTransition for the envs whose step ended; returns the TD errors.
        Backtest mode: State::newState of the next Backtester::_step (the greedy evaluation step; theta is only read);
        returns zeros, Backtester::_step computes no TD error."""
        out = (C.c_double * self.cfg.n_envs)()
        check(self.L.rlm_agent_update(self.h, out))
        return out

    # ---- shared policy (cfg.shared_policy = 1), SURVEY.md section 8e
    def shared_tick_accumulate(self):
        check(self.L.rlm_shared_tick_accumulate(self.h))

    def apply_dtheta(self):
        check(self.L.rlm_apply_dtheta(self.h))

    def dtheta_tensor(self):
        """Zero-copy torch view of the device dtheta buffer (for torch.distributed.all_reduce)."""
        import torch
        theta, dtheta, n = C.c_void_p(), C.c_void_p(), C.c_int64()
        check(self.L.rlm_device_ptrs(self.h, C.byref(theta), C.byref(dtheta), C.byref(n)))

        class _Buf:
            pass
        buf = _Buf()
        buf.__cuda_array_interface__ = {"shape": (n.value,), "typestr": "<f8", "data": (dtheta.value, False), "version": 2}
        t = torch.as_tensor(buf, device=torch.device("cuda", self.cfg.device))
        t._rlm_keepalive = self
        return t

    def records(self, env, cap=None):
        cap = self.cfg.record_cap if cap is None else cap
        out = (abi.StepRecord * cap)()
        n = C.c_int32(0)
        check(self.L.rlm_read_records(self.h, env, out, cap, C.byref(n)))
        return [out[i] for i in range(n.value)], out
