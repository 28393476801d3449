// oracle_market.cpp -- TEST INFRASTRUCTURE ONLY: Intraday::LoadData's market replacement for the CPU oracle.
//
// The reference builds the Market from the ticker each time it loads a day (Intraday::LoadData ->
// Market::make_market(symbol, venue), src/environment/intraday.cpp:141-150): a new market object with the venue's tick
// table and trading hours, while the agent, the books and the rolling windows carry on.  The oracle builds its market
// once, from the config (lob_oracle.cpp, lobo_env::init).  This file restates the replacement on top of the oracle's own
// source, compiled into a test-side library by tests/oracle_market.py; oracle/ itself stays as it is.
#include "lob_oracle.cpp"

extern "C" {

// the env's market becomes m (the config's venue block too, so that the env reads as created with m)
void lobo_set_market(lobo_env* e, const rlm_market* m) {
  rlm_config& c = e->c;
  c.n_bands = m->n_bands;
  for (int i = 0; i < RLM_MAX_BANDS; ++i) { c.band_px[i] = m->band_px[i]; c.band_ts[i] = m->band_ts[i]; }
  c.open_ms = m->open_ms;
  c.close_ms = m->close_ms;
  e->market.init(&c);  // a new Market (market.cpp:11-38): date and time start from 0
}

// env `env` of a shared-policy batch oracle
void lobo_batch_set_market(lobo_batch* b, int32_t env, const rlm_market* m) { lobo_set_market(b->envs[env], m); }

}
