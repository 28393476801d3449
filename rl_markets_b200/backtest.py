"""Evaluation outputs in the reference's file formats (SURVEY 8f rank 3).

  profit_log.csv  one row per Backtester step: Intraday::LogProfit (src/environment/intraday.cpp:437-451), header
                  from Backtester's ctor (src/experiment/serial.cpp:104-108).  Like upstream, the first two columns
                  carry market->date() and market->time() although the header calls them episode and step.
  test_stats.csv  Base::writeStats (src/environment/base.cpp:451-456).  Upstream opens the same path three times
                  with std::ofstream::out, so only the last writer (TradeStatistics, statistics.cpp:32-52)
                  survives; its four *_placed / *_cancelled counters are never incremented anywhere upstream.
  theta.bin       Agent::write_theta (src/rl/agent.cpp:176-181): MEMORY_SIZE raw doubles.

Numbers are printed with repr(), which -- like fmt's "{}" upstream -- is the shortest string that round-trips.
"""
import os

HEADER = "episode,step,action,position,midprice,spread,quoted_ask,quoted_bid,ask_level,bid_level,pnl_step,bandh_step"


def _num(x):
    if isinstance(x, float):
        return repr(int(x)) if x == int(x) and abs(x) < 1e15 else repr(x)
    return str(x)


def profit_rows(records, date):
    for r in records:
        yield ",".join(_num(v) for v in (date, r.time_ms, r.action, r.position, r.midprice, r.spread, r.ask_quote,
                                         r.bid_quote, r.ask_level, r.bid_level, r.pnl_step, r.bandh_step))


def test_stats_rows(records, market_sells, market_buys):
    """The eight rows Base::writeStats leaves in test_stats.csv.  trade_stats.{ask,bid}_transactions are copied from the
    books in Base::UpdateStats (base.cpp:412-417), which runs at the START of every step (base.cpp:278): what the file
    shows is the count after the last-but-one step, one step behind the books.  market_* are bumped where the market
    orders happen, the final ClearInventory included (base.cpp:339-349)."""
    lag = records[-2] if len(records) >= 2 else None
    return [("asks_placed", 0), ("bids_placed", 0), ("asks_cancelled", 0), ("bids_cancelled", 0),
            ("ask_transactions", lag.ask_transactions if lag else 0), ("bid_transactions", lag.bid_transactions if lag else 0),
            ("market_sells", market_sells), ("market_buys", market_buys)]


def write_logs(market, out_dir, env=0, date=20100104):
    """Write profit_log.csv / test_stats.csv / theta.bin for recorded env `env` of a handle in backtest mode
    (every step of the episode must be recorded: cfg.record_cap >= steps).  theta.bin is the policy env `env` ran under:
    its own, or the handle's one policy when cfg.shared_policy is set."""
    os.makedirs(out_dir, exist_ok=True)
    recs, _keep = market.records(env)
    paths = {k: os.path.join(out_dir, v) for k, v in
             (("profit_log", "profit_log.csv"), ("test_stats", "test_stats.csv"), ("theta", "theta.bin"))}
    with open(paths["profit_log"], "w") as f:
        f.write(HEADER + "\n")
        for row in profit_rows(recs, date):
            f.write(row + "\n")
    st = market.stats(env, 1)[0]
    with open(paths["test_stats"], "w") as f:
        for k, v in test_stats_rows(recs, st.market_sells, st.market_buys):
            f.write("%s,%d\n" % (k, v))
    with open(paths["theta"], "wb") as f:
        f.write(bytes(market.theta(0 if market.cfg.shared_policy else env)))
    return paths
