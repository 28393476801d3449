"""Reference-format CSV pair -> packed rlm_tick_msg stream (SURVEY.md section 8f rank 1).

The parser lives in the library (rl_markets_b200/csrc/rlm_ingest.cpp, C ABI rlm_ingest_csv in include/rlm.h): it
restates the reference's data layer -- row filtering and number parsing of data::basic (src/data/basic.cpp:20-202), print
aggregation of Streamer::LoadUntil (src/data/streamer.cpp:57-81), row grouping of Intraday::UpdateBookProfiles
(src/environment/intraday.cpp:274-313) -- and represents what round 1 rejected: depth rows that share a timestamp or
follow an invalid book state (RLM_TICK_PARTIAL) and ticks with more than four distinct print prices (RLM_TICK_TX_MORE).
This module is the Python face of it."""
import glob as _glob
import os

from . import lib


def file_sample(md_dir, tas_dir, symbols):
    """get_file_sample (include/utilities/files.h:39-76): the (symbol, md csv, tas csv) tuples the reference's driver
    trains on.  For every symbol every `<md_dir>/<symbol>/*.csv` (glob order) whose partner exists; the partner's path is
    the md path with the md_dir prefix swapped for tas_dir and then -- at the OFFSET where "md_" first occurs in the md
    path, applied to the tas path as upstream does -- the two characters after that offset's first replaced by "tas"
    (so ".../xmd_2010.csv" -> ".../xmtas2010.csv": the upstream rule keeps the 'm' and swallows "d_"; with directory
    names of different lengths the offset lands elsewhere: reproduced, not fixed).  Raises like the reference on a
    missing symbol directory or an md file without "md_" in its path."""
    out = []
    for s in symbols:
        md_s, tas_s = md_dir + "/" + s, tas_dir + "/" + s
        if not os.path.exists(md_s):
            raise RuntimeError("No such directory: " + md_s)
        if not os.path.exists(tas_s):
            raise RuntimeError("No such directory: " + tas_s)
        for f in sorted(_glob.glob(_glob.escape(md_s) + "/*.csv")):
            tf = tas_dir + f[len(md_dir):]
            loc = f.find("md_")
            if loc < 0:
                raise RuntimeError("Unexpected file name: " + f)
            tf = tf[:loc + 1] + "tas" + tf[loc + 3:]
            if os.access(tf, os.F_OK):
                out.append((s, f, tf))
    return out


def sample_window(md_dir, tas_dir, symbol, search_patterns):
    """get_sample_window (files.h:78-108): per pattern the FIRST md and the FIRST tas file matching `*<pattern>*.csv`
    (the evaluation days of main.cpp); the two lists must have equal length."""
    md_s, tas_s = md_dir + "/" + symbol, tas_dir + "/" + symbol
    if not os.path.exists(md_s):
        raise RuntimeError("No such directory: " + md_s)
    if not os.path.exists(tas_s):
        raise RuntimeError("No such directory: " + tas_s)
    out = []
    for p in search_patterns:
        md_files = sorted(_glob.glob(_glob.escape(md_s) + "/*" + p + "*.csv"))
        tas_files = sorted(_glob.glob(_glob.escape(tas_s) + "/*" + p + "*.csv"))
        if len(md_files) != len(tas_files):
            raise RuntimeError("No matching files for MD and TAS.")
        out.append((symbol, md_files[0], tas_files[0]))
    return out


def csv_pair_to_ticks(md_path, tas_path):
    """Returns (ctypes array of TickMsg, number of messages, number of market ticks they make up)."""
    return lib.ingest_csv(md_path, tas_path)


def day_library(samples):
    """The (symbol, md csv, tas csv) tuples of file_sample / sample_window -> (msgs, offsets) for BatchedMarket.load_days:
    every pair through rlm_ingest_csv, the message streams one after the other, offsets[d] = first message of day d and
    offsets[-1] = the total."""
    import ctypes as C
    from . import abi
    days = [lib.ingest_csv(md, tas) for _symbol, md, tas in samples]
    offsets = [0]
    for _msgs, n, _ticks in days:
        offsets.append(offsets[-1] + n)
    out = (abi.TickMsg * max(offsets[-1], 1))()
    size = C.sizeof(abi.TickMsg)
    for (msgs, n, _ticks), off in zip(days, offsets):
        C.memmove(C.addressof(out) + off * size, msgs, n * size)
    return out, offsets


def day_markets(samples):
    """The (symbol, md csv, tas csv) tuples of file_sample / sample_window -> (markets, day_market) for
    BatchedMarket.set_day_markets: day d runs under markets[day_market[d]], its symbol's market (config.market), as
    Intraday::LoadData builds it from the ticker (src/environment/intraday.cpp:141-150).  Markets are deduplicated by tick
    table and trading hours, in first-seen order."""
    from . import config
    markets, day_market = [], []
    for symbol, _md, _tas in samples:
        m = config.market(symbol)
        k = next((i for i, o in enumerate(markets) if config.same_market(o, m)), None)
        if k is None:
            k = len(markets)
            markets.append(m)
        day_market.append(k)
    return markets, day_market


def load_day(market, md_path, tas_path):
    """Intraday::LoadData (src/environment/intraday.cpp:141-150) for every env of a STREAM-source handle: the same day for
    all of them.  Returns the number of message slots to pass to run_ticks."""
    import ctypes as C
    from . import abi
    msgs, n, _ticks = lib.ingest_csv(md_path, tas_path)
    B = market.cfg.n_envs
    wide = (abi.TickMsg * (n * B))()
    for t in range(n):
        for b in range(B):
            wide[t * B + b] = msgs[t]
    market.load_ticks(wide, n)
    return n
