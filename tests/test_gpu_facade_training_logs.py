"""The class surface's training logs: examples/serial_driver --train-log-dir D, written against include/rlm_facade.hpp
(rl::Agent(session, D) and experiment::serial::Learner(env, D)), must leave D/model_log.csv and D/training_log.csv equal
byte for byte to the files the reference writes into its output_dir (tests/golden/tl_*, tools/make_golden.py
--training-logs): a synthetic day and a venue CSV pair on the tape source."""
import os
import subprocess
import tempfile

import pytest

import golden_util as G
import test_training_logs as TL

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "examples", "serial_driver")
_VENUE = {c["name"]: c for c in G.venue_manifest()}


def _files(d):
    return tuple(open(os.path.join(d, n)).read() for n in ("model_log.csv", "training_log.csv"))


def _want(c):
    return TL.fixture(c, "model_log"), TL.fixture(c, "training_log")


def test_synthetic_day():
    c = TL.case("tl_q_learn_eps")
    day = c["days"][0]
    assert c["algo"] == "q_learn" and set(c["over"]) == {"policy.eps_T"} and len(c["days"]) == 1
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call([DRIVER, "--episodes", str(c["episodes"]), "--algo", c["algo"], "--memory-size", str(c["M"]),
                               "--open-ticks", str(day["open_ticks"]), "--flow-seed", str(day["flow_seed"]),
                               "--eps-T", str(c["over"]["policy.eps_T"]), "--env", str(c["env"]), "--train-log-dir", d],
                              stdout=subprocess.DEVNULL)
        assert _files(d) == _want(c)


def test_venue_day_on_the_tape_source():
    c = TL.case("tl_venue_aal")
    assert c["algo"] == "q_learn" and not c["over"] and len(c["days"]) == 1
    with tempfile.TemporaryDirectory() as d:
        md, tas = G.venue_day(_VENUE[c["days"][0]["venue"]], d)
        logs = os.path.join(d, "logs")
        os.mkdir(logs)
        subprocess.check_call([DRIVER, "--md", md, "--tas", tas, "--episodes", str(c["episodes"]), "--algo", c["algo"],
                               "--memory-size", str(c["M"]), "--env", str(c["env"]), "--train-log-dir", logs],
                              stdout=subprocess.DEVNULL)
        assert _files(logs) == _want(c)


def test_no_log_dir_writes_nothing():
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call([DRIVER, "--episodes", "1", "--memory-size", "4096"], cwd=d, stdout=subprocess.DEVNULL)
        assert os.listdir(d) == []
