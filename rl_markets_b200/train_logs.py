"""Training outputs in the reference's file formats (logging.log_learning, config/example.yaml).

  model_log.csv     Agent::HandleTransition (src/rl/agent.cpp:86-101): on every 1000th update one line, the mean
                    |TD error| of those 1000 updates (_agg_delta / 1000).  No header (the logger is created without one,
                    agent.cpp:52-59).  The counter runs across episodes.
  training_log.csv  Learner::RunEpisode (src/experiment/serial.cpp:42-49,72-94): the header of Learner's ctor, then one
                    row per episode after HandleTerminal -- the incremented episode counter, Intraday::getEpisodeId()
                    (to_string(init_date), intraday.cpp:160), episode reward and P&L, the episode's _step_counter and
                    policy->descr() (eps / tau / 0, read after HandleTerminal has decayed it).

Both loggers use the pattern "%v" (main.cpp:254), so a line is the formatted message alone; numbers go through
backtest._num, the same rendering of fmt's "{}" as profit_log.csv.  One reference process writes one pair of files: on
the device that is one env of a handle (TrainingLogs(market, out_dir, env)).
"""
import os

from .backtest import _num

MODEL_LOG = "model_log.csv"
TRAINING_LOG = "training_log.csv"
TRAINING_HEADER = "episode,episode_id,reward,pnl,n_steps,epsilon"


def model_log_lines(values):
    """The lines of model_log.csv for logged values (floats)."""
    return [_num(float(v)) for v in values]


def training_log_line(episode, episode_id, reward, pnl, n_steps, descr):
    """One row of training_log.csv: spdlog's "{},{},{},{},{},{}" of serial.cpp:81-88.  `episode` is the counter after
    the increment (episode e of handle_terminal(e) is row e + 1)."""
    return ",".join((str(int(episode)), str(episode_id), _num(float(reward)), _num(float(pnl)), str(int(n_steps)), _num(float(descr))))


def model_log_values(deltas, agg=0.0, count=0):
    """HandleTransition's arithmetic on a sequence of TD errors: returns (logged values, agg, count) -- the reference's
    sequential sum of abs(delta), divided by 1000 on every 1000th update.  Pass agg / count back in to continue."""
    out = []
    for d in deltas:
        agg += abs(d)
        count += 1
        if count == 1000:
            out.append(agg / 1000.0)
            agg, count = 0.0, 0
    return out, agg, count


class TrainingLogs:
    """model_log.csv and training_log.csv of env `env` of a BatchedMarket, as the reference process that env stands for
    writes them into its output_dir.  Turns the handle's model_log on (market.set_model_log(cap_rows)) unless it is on
    already; for the files to equal the reference's, create this right after the handle.  Per episode e:

        run until every env is terminal; market.handle_terminal(e); logs.episode_end(e, episode_id); market.reset()

    episode_id is what Intraday::getEpisodeId() returns: the date (YYYYMMDD) of the day the episode ran on."""

    def __init__(self, market, out_dir, env=0, cap_rows=4096):
        self.market, self.env = market, env
        if not getattr(market, "_mlog_cap", 0):
            market.set_model_log(cap_rows)
        os.makedirs(out_dir, exist_ok=True)
        self.paths = {"model_log": os.path.join(out_dir, MODEL_LOG), "training_log": os.path.join(out_dir, TRAINING_LOG)}
        open(self.paths["model_log"], "w").close()
        with open(self.paths["training_log"], "w") as f:
            f.write(TRAINING_HEADER + "\n")

    def flush(self):
        """Append the env's model_log values logged since the last read."""
        vals = self.market.model_log(self.env, 1)[0]
        if vals:
            with open(self.paths["model_log"], "a") as f:
                f.write("".join(v + "\n" for v in model_log_lines(vals)))

    def episode_end(self, episode, episode_id):
        """The training_log row of episode `episode` (the argument of the handle_terminal just made), then flush()."""
        st = self.market.stats(self.env, 1)[0]
        row = training_log_line(episode + 1, episode_id, st.episode_reward, st.episode_pnl, st.steps, self.market.policy_descr())
        with open(self.paths["training_log"], "a") as f:
            f.write(row + "\n")
        self.flush()
