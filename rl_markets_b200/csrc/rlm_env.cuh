// rlm_env.cuh -- scalar (one-lane) market logic of the batched LOB environment.
//
// These functions are executed by lane 0 of the warp that owns the env, on the
// env record staged in shared memory.  They restate, for ONE agent order per
// side (ORDER_LIMIT == 1, src/environment/base.cpp:21), the reference's
//   market::Order            src/market/order.cpp:34-118
//   market::Book/Ask/Bid     src/market/book.cpp:50-141,249-261,382-539
//   BookUtils                src/market/book.cpp:550-625
//   market::Market           src/market/market.cpp:67-138
//   environment::RiskManager src/environment/risk_manager.cpp:26-113
//   environment::Base        src/environment/base.cpp:166-237,254-349,412-442
//   environment::Intraday    src/environment/intraday.cpp:64-82,163-272,315-409
// keeping the reference's fp64 operation order (compiled with -fmad=false) so
// that integer book state is bit-exact and fp64 state is bitwise equal too.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include "rlm_types.h"

__constant__ DevParams P;
__constant__ DevMarkets PM;

#define LLMIN ((long long)0x8000000000000000ull)
// per-level loops of the book code: unrolled (five copies, independent loads in flight) or rolled (a fifth of the code;
// instruction fetch is this kernel's largest stall).  Unrolled is the default; RLM_ROLL_LEVELS builds the rolled form
#ifdef RLM_ROLL_LEVELS
#define LEVEL_UNROLL _Pragma("unroll 1")
#else
#define LEVEL_UNROLL _Pragma("unroll")
#endif

// ---------------------------------------------------------------- utilities/comparison.h:13-16
__device__ __forceinline__ double pkey(double p) { return rint(p * 10000.0); }

// x86-64 cvttsd2si: out-of-range and NaN give the "integer indefinite" value (SURVEY Appendix A5);
// CUDA's cvt.rzi.s64.f64 would saturate instead.
__device__ __forceinline__ long long d2ll_x86(double d) {
  if (!(d >= -9223372036854775808.0 && d < 9223372036854775808.0)) return LLMIN;
  return (long long)d;
}

// ---------------------------------------------------------------- market::Market
// Which Market a tick reads.  The config's lives in the __constant__ block (P.venue).  A tape day with a market of its own
// (rlm_set_day_markets: Intraday::LoadData building the ticker's market, intraday.cpp:141-150) hands the env's VenueD
// from global memory as an EnvMarket.  Every function that reads the market takes it as a trailing parameter pack: empty
// on the config's path, which so compiles to the code it had before day markets existed.
struct EnvMarket { const VenueD* v; };
__device__ __forceinline__ const VenueD& venue_of() { return P.venue; }
__device__ __forceinline__ const VenueD& venue_of(EnvMarket m) { return *m.v; }

static_assert((RLM_MAX_BANDS & (RLM_MAX_BANDS - 1)) == 0, "the band search halves RLM_MAX_BANDS");
// Market::ToTicks (market.cpp:78-102).  Bands below the one containing `price` contribute a
// price-independent chain of truncating `int += double` steps, precomputed on the host
// (VenueD::cum_full); the loop below is the reference loop entered at that band.
// band_hint (optional): in/out, the band of the caller's previous conversion -- prices stay inside one band for hours, so
// two comparisons usually replace the five dependent look-ups of the search.  A band whose tick size is a power of two
// (VenueD::inv_ts != 0) is divided by multiplying with the exact reciprocal: the same IEEE result without the fp64
// division sequence.
__device__ __forceinline__ int to_ticks_in(const VenueD& V, double price, int* err, int* band_hint) {
  if (price < V.px[0]) { *err |= ERR_TICK_RANGE; return 0; }
  int k = 0;  // band containing price = last band start <= price (px[i >= n] = +inf, px[0] <= price)
  const int hk = band_hint ? *band_hint : -1;
  if ((unsigned)hk < (unsigned)(RLM_MAX_BANDS - 1) && !(price < V.px[hk]) && price < V.px[hk + 1]) {
    k = hk;
  } else {  // binary search
#pragma unroll
    for (int step = RLM_MAX_BANDS / 2; step >= 1; step >>= 1)
      if (!(price < V.px[k + step])) k += step;
    if (band_hint) *band_hint = k;
  }
  int ticks = V.cum_full[k];
  double tsp = V.ts[k];  // tick_size(price) = band containing price (market.cpp:130-138)
  int it = k;
#pragma unroll 1
  while (it < V.n && price + V.ts[it] / 2.0 > V.px[it]) {
    double ub;
    if (it == V.n - 1 || price < V.px[it + 1]) ub = price + tsp / 2.0;
    else ub = V.px[it + 1];
    const double inv = V.inv_ts[it];
    const double q = (inv != 0.0) ? (ub - V.px[it]) * inv : (ub - V.px[it]) / V.ts[it];
    ticks = (int)((double)ticks + q);  // int += double
    ++it;
  }
  return ticks;
}

__device__ __noinline__ int to_ticks(double price, int* err, int* band_hint = nullptr) { return to_ticks_in(P.venue, price, err, band_hint); }
__device__ __noinline__ int to_ticks(EnvMarket m, double price, int* err, int* band_hint = nullptr) { return to_ticks_in(*m.v, price, err, band_hint); }

// Market::ToPrice (market.cpp:104-128), same prefix trick on Market::tts_.
__device__ __forceinline__ double to_price_in(const VenueD& V, int ticks, int* err) {
  if (ticks < V.tts_tick[0]) { *err |= ERR_TICK_RANGE; return 0.0; }
  if (!(ticks > V.tts_tick[0])) return 0.0;
  int k = 0;  // last tts_ key <= ticks (tts_tick[i >= n] = INT_MAX)
#pragma unroll
  for (int step = RLM_MAX_BANDS / 2; step >= 1; step >>= 1)
    if (ticks >= V.tts_tick[k + step]) k += step;
  // bands 0..k-1 fully traversed; band k partially (or exactly to its end when ticks == next key)
  double price = V.cum_price[k];
  if (ticks > V.tts_tick[k]) price += ((double)ticks - (double)V.tts_tick[k]) * V.ts[k];
  return price;
}

__device__ __noinline__ double to_price(int ticks, int* err) { return to_price_in(P.venue, ticks, err); }
__device__ __noinline__ double to_price(EnvMarket m, int ticks, int* err) { return to_price_in(*m.v, ticks, err); }

template <class... M>
__device__ __forceinline__ bool market_is_open(const EnvHdr& e, M... mk) {  // market.cpp:67-70
  const VenueD& V = venue_of(mk...);
  return ((long long)e.time_ms > V.open_lo) && ((long long)e.time_ms < V.close_hi);
}
template <class... M>
__device__ __forceinline__ bool is_terminal(const EnvHdr& e, M... mk) {  // intraday.cpp:152-157
  return (!market_is_open(e, mk...)) || ((e.last_date != 0) && (e.date != e.last_date));
}

// ---------------------------------------------------------------- market::Order
__device__ __forceinline__ long long ord_remaining(const OrderD& o) {  // order.cpp:34-37
  long long r = o.size - o.executed;
  return r > 0 ? r : 0;
}
__device__ __forceinline__ bool ord_is_executed(const OrderD& o) { return o.executed >= o.size; }  // :49-52

__device__ __noinline__ long long ord_do_transaction(OrderD& o, long long volume) {  // order.cpp:54-82
  o.transactions += (int)volume;
  long long remaining_volume = volume - o.q_head;
  if (remaining_volume > 0) {
    o.q_head = 0;
    if (ord_remaining(o) <= remaining_volume) {
      o.executed = o.size;
      remaining_volume -= o.size;
    } else {
      o.executed += remaining_volume;
      remaining_volume = 0;
    }
  } else {
    o.q_head -= volume;
  }
  return remaining_volume > 0 ? remaining_volume : 0;
}

__device__ __noinline__ void ord_do_cancellation(OrderD& o, long long volume) {  // order.cpp:84-107
  if (o.q_tail == 0) {
    o.q_head -= volume;
  } else {
    double total = (double)(o.q_head + o.q_tail);
    // `long -= double`: long -> double, subtract, double -> long
    o.q_head = d2ll_x86((double)o.q_head - ceil((double)(volume * o.q_head) / total));
    o.q_tail = d2ll_x86((double)o.q_tail - floor((double)(volume * o.q_tail) / total));
  }
  if (o.q_head < 0) {
    o.q_tail = (long long)((unsigned long long)o.q_tail + (unsigned long long)o.q_head);
    o.q_head = 0;
  }
  if (o.q_tail < 0) o.q_tail = 0;
}

// ---------------------------------------------------------------- market::Book
__device__ long long side_volume(const SideD& s, double price) {  // book.cpp:208-214
  if (!s.has_cur) return 0;
  double k = pkey(price);
  long long v = 0;
  LEVEL_UNROLL
  for (int l = 0; l < RLM_DEPTH; ++l)
    if (pkey(s.px[l]) == k) v = s.vol[l];
  return v;
}
__device__ long long side_last_volume(const SideD& s, double price) {  // book.cpp:216-222
  if (!s.has_last) return 0;
  double k = pkey(price);
  long long v = 0;
  LEVEL_UNROLL
  for (int l = 0; l < RLM_DEPTH; ++l)
    if (pkey(s.last_px[l]) == k) v = s.last_vol[l];
  return v;
}

__device__ __noinline__ void side_reset(SideD& s) {  // book.cpp:143-160
  s.n_transacted = 0; s.obs_value = 0.0; s.obs_volume = 0;
  s.total_vol = 0; s.last_total_vol = 0;
  for (int l = 0; l < RLM_DEPTH; ++l) { s.px[l] = 0.0; s.last_px[l] = 0.0; s.vol[l] = 0; s.last_vol[l] = 0; }
  s.has_cur = 0; s.has_last = 0;
  s.ord.live = 0;
}

// Book::PlaceOrder (book.cpp:249-261) after RiskManager::PlaceOrder's CancelWorst
// (risk_manager.cpp:61-99): with one order per side the old order is always replaced.
__device__ __noinline__ void side_replace_order(SideD& s, double price, long long size, int* err) {
  if (price <= 0 || size <= 0) { *err |= ERR_BAD_PRICE; s.ord.live = 0; return; }  // order.cpp:22-27
  OrderD& o = s.ord;
  o.live = 1; o.price = price; o.size = size;
  o.q_head = side_volume(s, price);
  o.q_tail = 0; o.executed = 0; o.transactions = 0; o.initial_queue = o.q_head;
}

// Book::UpdateOrder (book.cpp:101-141)
__device__ __noinline__ void side_update_order(SideD& s, long long transaction_volume) {
  OrderD& o = s.ord;
  if (!o.live) return;
  if (ord_is_executed(o)) { o.live = 0; return; }
  long long lv = side_last_volume(s, o.price);
  if (lv == 0) return;
  long long v = side_volume(s, o.price);
  if (v == 0) { o.q_head = 0; o.q_tail = 0; return; }
  long long vol_diff = lv - v;
  if (vol_diff >= 0) {
    long long cancelled = vol_diff - transaction_volume;
    if (cancelled > 0) ord_do_cancellation(o, cancelled);
  } else {
    o.q_tail += vol_diff;  // addVolumeBehind with a negative volume (SURVEY Appendix A4)
  }
}

// Book::StashState (book.cpp:50-55)
__device__ __forceinline__ void side_stash(SideD& s) {
  LEVEL_UNROLL
  for (int l = 0; l < RLM_DEPTH; ++l) { s.last_px[l] = s.px[l]; s.last_vol[l] = s.vol[l]; }
  s.has_last = s.has_cur;
  s.last_total_vol = s.total_vol;
}
// Book::ApplyChanges for one depth row (book.cpp:63-99).  px/vol: the side's 5 levels, best first (the stream contract);
// tpx/tvol/n_tx: the tick's aggregated prints (the `transactions` map handed through UpdateBookProfiles).
__device__ __forceinline__ void side_apply_row(SideD& s, const float* px, const int* vol, const float* tpx, const int* tvol, int n_tx, int* err) {
  long long tv = s.total_vol;
  LEVEL_UNROLL
  for (int l = 0; l < RLM_DEPTH; ++l) {
    double p = (double)px[l];
    int v = vol[l];
    if (p <= 0.0 || v <= 0) *err |= ERR_BAD_PRICE;
    s.px[l] = p; s.vol[l] = v;
    tv += v;
  }
  s.total_vol = tv;
  s.has_cur = 1;
  if (s.ord.live) {
    // transactions.find(order price) by comparator key (book.cpp:94-95)
    long long t = 0;
    double k = pkey(s.ord.price);
    for (int i = 0; i < n_tx; ++i)
      if (pkey((double)tpx[i]) == k) t = tvol[i];
    side_update_order(s, t);
  }
}
// Book::StashState + Book::ApplyChanges for one depth row = one tick (the synthetic flow's contract)
__device__ __noinline__ void side_apply_changes(SideD& s, const float* px, const int* vol, const rlm_tick_msg& m, int* err) {
  side_stash(s);
  side_apply_row(s, px, vol, m.tx_px, m.tx_vol, m.n_tx, err);
}

struct Fill { long long volume; double proxy, value; };

// AskBook::ApplyTransactions (book.cpp:382-427) / BidBook::ApplyTransactions (:467-510) over n aggregated prints
template <bool IS_ASK>
__device__ __forceinline__ Fill side_apply_transactions_n(SideD& s, const float* tpx, const int* tvol, int n, double ref) {
  s.obs_value = 0.0;
  s.obs_volume = 0;
  Fill f; f.volume = 0; f.proxy = 0.0; f.value = 0.0;
  OrderD& o = s.ord;
  for (int k = 0; k < n; ++k) {
    const int i = IS_ASK ? k : n - 1 - k;
    const double tp = (double)tpx[i];
    if (IS_ASK ? (tp < ref) : (tp > ref)) continue;
    long long vol = tvol[i];
    s.obs_value += tp * (double)vol;
    s.obs_volume += vol;
    while (o.live && (IS_ASK ? (o.price <= tp) : (o.price >= tp))) {
      long long rem0 = ord_remaining(o);
      vol = ord_do_transaction(o, vol);
      long long exec = rem0 - ord_remaining(o);
      if (IS_ASK) {
        f.volume -= exec;
        f.proxy += (o.price - ref) * (double)exec;
        f.value += o.price * (double)exec;
      } else {
        f.volume += exec;
        f.proxy += (ref - o.price) * (double)exec;
        f.value -= o.price * (double)exec;
      }
      if (ord_is_executed(o)) { o.live = 0; s.n_transacted++; }
      if (vol <= 0) break;
    }
  }
  return f;
}
template <bool IS_ASK>
__device__ __noinline__ Fill side_apply_transactions(SideD& s, const rlm_tick_msg& m, double ref, bool use_tx) {
  return side_apply_transactions_n<IS_ASK>(s, m.tx_px, m.tx_vol, use_tx ? m.n_tx : 0, ref);
}

// AskBook/BidBook::WalkTheBook (book.cpp:429-456,512-539)
template <bool IS_ASK>
__device__ __noinline__ Fill side_walk(SideD& s, double ref, long long size) {
  Fill f; f.volume = 0; f.proxy = 0.0; f.value = 0.0;
  long long abs_size = size < 0 ? -size : size;
  if (abs_size > s.total_vol) return f;
  long long executed = 0;
  for (int l = 0; l < RLM_DEPTH; ++l) {  // levels map iterates best-first
    long long lvol = s.vol[l];
    long long l_ex = lvol < (abs_size - executed) ? lvol : (abs_size - executed);
    executed += l_ex;
    f.proxy -= (double)l_ex * fabs(s.px[l] - ref);
    if (IS_ASK) f.value -= (double)l_ex * s.px[l];
    else f.value += (double)l_ex * s.px[l];
    if (executed >= abs_size) { s.n_transacted++; break; }
  }
  f.volume = IS_ASK ? executed : -executed;
  return f;
}

// include/market/measures.h
__device__ __forceinline__ double m_midprice(const EnvHdr& e) { return (e.side[0].px[0] + e.side[1].px[0]) / 2.0; }
__device__ __forceinline__ double m_last_midprice(const EnvHdr& e) { return (e.side[0].last_px[0] + e.side[1].last_px[0]) / 2.0; }
__device__ __forceinline__ double m_spread(const EnvHdr& e) { return e.side[0].px[0] - e.side[1].px[0]; }
__device__ __forceinline__ double m_microprice(const EnvHdr& e) {  // measures.h:39-53 (cumulative volumes, A2)
  double ap = e.side[0].px[0], bp = e.side[1].px[0];
  long long av = e.side[0].total_vol, bv = e.side[1].total_vol;
  double div = (double)(av + bv);
  double mpm_a = (double)av * bp;
  double mpm_b = ap * (double)bv;
  return (mpm_a + mpm_b) / div;
}

// BookUtils::HandleAdverseSelection (book.cpp:550-592)
__device__ __noinline__ Fill adverse_selection(EnvHdr& e) {
  SideD& ask = e.side[0];
  SideD& bid = e.side[1];
  const double bap = ask.px[0], bbp = bid.px[0], rp = m_last_midprice(e);
  Fill f; f.volume = 0; f.proxy = 0.0; f.value = 0.0;
  if (ask.ord.live && ask.ord.price <= bbp) {
    long long rem = ord_remaining(ask.ord);
    f.volume -= rem;
    f.proxy += (double)rem * (ask.ord.price - rp);
    f.value += (double)rem * ask.ord.price;
    ask.ord.live = 0;
    ask.n_transacted++;
  }
  if (bid.ord.live && bid.ord.price >= bap) {
    long long rem = ord_remaining(bid.ord);
    f.volume += rem;
    f.proxy += (double)rem * (rp - bid.ord.price);
    f.value -= (double)rem * bid.ord.price;
    bid.ord.live = 0;
    bid.n_transacted++;
  }
  return f;
}

// ---------------------------------------------------------------- RiskManager / Base / Intraday
__device__ __forceinline__ void check_orders(EnvHdr& e) {  // risk_manager.cpp:26-32
  if (e.position >= P.pos_ub) e.side[1].ord.live = 0;
  else if (e.position <= P.pos_lb) e.side[0].ord.live = 0;
}

// window accessors (rings live right behind the header)
__device__ __forceinline__ double win_front(const EnvHdr& e, const double* ring, int w) {
  int ws = P.win_size[w];
  int i = e.w_head[w] - 1; if (i < 0) i += ws;
  return ring[P.win_off[w] + i];
}
__device__ __forceinline__ double win_back(const EnvHdr& e, const double* ring, int w) {
  int i = (e.w_count[w] == P.win_size[w]) ? e.w_head[w] : 0;
  return ring[P.win_off[w] + i];
}
__device__ __forceinline__ double win_std(const EnvHdr& e, int w) {  // accumulators.cpp:117-131
  double v = e.w_s[w] / (double)((unsigned long long)((long long)e.w_count[w] - 1));
  return v > 0 ? sqrt(v) : 0.0;
}

// Base::getReward (base.cpp:166-237)
__device__ __noinline__ double get_reward(const EnvHdr& e) {
  double r = 0.0;
  long long ap = e.position < 0 ? -e.position : e.position;
  int abs_pos = (int)ap;
  switch (P.reward_measure) {
    case RLM_REWARD_NONE: break;
    case RLM_REWARD_PNL: r = e.pnl_step; break;
    case RLM_REWARD_PNL_DAMPED: r = e.pnl_step - (double)P.damping * fmax(0.0, e.momentum_pnl_step); break;
    case RLM_REWARD_SPREAD: r = e.pnl_step / e.w_mean[W_SPREAD]; break;
    case RLM_REWARD_NORMED:
      if (!(e.w_count[W_PNLUP] == P.win_size[W_PNLUP] && e.w_count[W_PNLDN] == P.win_size[W_PNLDN])) r = 0.0;
      else {
        double u = e.w_mean[W_PNLUP], d = e.w_mean[W_PNLDN];
        double su = win_std(e, W_PNLUP), sd = win_std(e, W_PNLDN);
        double numer = (u * sd - d * su), denom = (su + sd);
        if (isnan(numer) || isinf(numer)) numer = 0.0;
        if (isnan(denom) || isinf(denom)) denom = 0.0;
        r = (fabs(denom) < 1e-5) ? numer : (numer / denom);
      }
      break;
    case RLM_REWARD_LOVOL: r = (double)e.lo_vol_step; break;
    case RLM_REWARD_MM_LINEAR: r = (double)(-P.pos_weight * (float)abs_pos); r += (double)P.pnl_weight * e.pnl_step; break;
    case RLM_REWARD_MM_EXP:  // libm exp/pow: tolerance parity only (documented in DESIGN.md)
      r = -pow(1.0 - exp((double)(P.pos_weight * (float)abs_pos)), 2.0); r += (double)P.pnl_weight * e.pnl_step; break;
    case RLM_REWARD_MM_DIV:
      if (e.pnl_step > 0) r = e.pnl_step / fmax(1.0, (double)abs_pos);
      else r = e.pnl_step;
      break;
  }
  return r * 100.0;
}

// Base::ClearInventory + RiskManager::ClearInventory/MarketOrder + BookUtils::MarketOrder
// (base.cpp:339-349, risk_manager.cpp:101-113, book.cpp:594-610)
__device__ __noinline__ void clear_inventory(EnvHdr& e) {
  long long size = -e.position;
  Fill f; f.volume = 0; f.proxy = 0.0; f.value = 0.0;
  double mip = m_midprice(e);
  if (size > 0) f = side_walk<true>(e.side[0], mip, size);
  else if (size < 0) f = side_walk<false>(e.side[1], mip, size);
  e.position += f.volume;
  e.pnl_step += f.proxy;
  e.lo_vol_step += (int)(f.volume < 0 ? -f.volume : f.volume);
  e.ep_pnl += f.value;
  if (f.volume > 0) e.market_buys++;
  else if (f.volume < 0) e.market_sells++;
}

// Intraday::l2p_ + _place_orders (intraday.cpp:64-82,163-173)
template <class... M>
__device__ __noinline__ void place_orders(EnvHdr& e, int al, int bl, M... mk) {
  e.ask_level = al; e.bid_level = bl;
  if (P.l2p_book) {
    e.ask_quote = to_price(mk..., to_ticks(mk..., e.side[0].px[0], &e.err, &e.tk_band) + al, &e.err);
    e.bid_quote = to_price(mk..., to_ticks(mk..., e.side[1].px[0], &e.err, &e.tk_band) - bl, &e.err);
  } else {
    double tp = e.tp_val, half_spd = fmax(0.0, e.w_mean[W_SPREAD] / 2.0);
    e.ask_quote = to_price(mk..., to_ticks(mk..., tp + (double)al * half_spd, &e.err, &e.tk_band), &e.err);
    e.bid_quote = to_price(mk..., to_ticks(mk..., tp - (double)bl * half_spd, &e.err, &e.tk_band), &e.err);
  }
  side_replace_order(e.side[0], e.ask_quote, P.order_size, &e.err);
  side_replace_order(e.side[1], e.bid_quote, P.order_size, &e.err);
}

// Intraday::DoAction (intraday.cpp:175-220): action -> (ask_level, bid_level)
template <class... M>
__device__ __noinline__ void do_action(EnvHdr& e, int action, M... mk) {
  int al, bl;
  switch (action) {
    case 0: al = 1; bl = 1; break;
    case 1: clear_inventory(e); al = e.ask_level; bl = e.bid_level; break;
    case 2: al = 2; bl = 2; break;
    case 3: al = 3; bl = 3; break;
    case 4: al = 0; bl = 2; break;
    case 5: al = 2; bl = 0; break;
    case 6: al = 1; bl = 4; break;
    case 7: al = 4; bl = 1; break;
    case 8: al = 5; bl = 5; break;
    default: return;
  }
  place_orders(e, al, bl, mk...);
}

// Base::UpdateStats (base.cpp:412-442)
__device__ __noinline__ void update_stats(EnvHdr& e) {
  e.ts_total++;
  bool has_ask = e.side[0].ord.live, has_bid = e.side[1].ord.live;
  if (has_ask) e.ts_ask++;
  if (has_bid) e.ts_bid++;
  if (has_ask && has_bid) e.ts_both++;
  if (e.position != 0) e.ts_pos++;
  if (e.position > 0) e.ts_long++;
  else if (e.position < 0) e.ts_short++;
}

// Intraday::UpdateBookProfiles for one row (intraday.cpp:274-313)
__device__ __noinline__ void update_book_profiles(EnvHdr& e, const rlm_tick_msg& m) {
  e.last_date = e.date;
  e.date = m.date;
  e.time_ms = m.time_ms;
  side_apply_changes(e.side[0], m.ask_px, m.ask_vol, m, &e.err);
  side_apply_changes(e.side[1], m.bid_px, m.bid_vol, m, &e.err);
  if (e.side[0].has_last && e.side[1].has_last && !(pkey(e.side[0].last_px[0]) == 0.0) && !(pkey(e.side[1].last_px[0]) == 0.0)) {
    double mp = m_midprice(e);  // BookUtils::IsValidState (book.cpp:612-625); the reference would swallow further rows
    bool ok = (m_spread(e) >= 0.0) && (mp > 0.0) && (fabs(mp - m_last_midprice(e)) < mp);
    if (!ok) e.err |= ERR_INVALID_STATE;
  }
}

// second half of NextState (intraday.cpp:242-269): adverse selection, P&L / position book-keeping, the
// eight values to push into the rolling windows
template <class... M>
__device__ __noinline__ void next_state_tail(EnvHdr& e, const Fill& au, const Fill& bu, double* pushv, M... mk) {
  Fill as = adverse_selection(e);
  e.pnl_step += au.proxy + bu.proxy + as.proxy;
  long long asabs = as.volume < 0 ? -as.volume : as.volume;
  e.lo_vol_step += (int)(bu.volume - au.volume + asabs);
  e.ep_pnl += au.value + bu.value + as.value;
  e.position += bu.volume + au.volume + as.volume;  // RiskManager::Update (risk_manager.cpp:34-39)
  check_orders(e);
  double mid = m_midprice(e);
  // (memo: ToTicks is a pure function of the price; a zero-initialised memo can only match mid == 0, which is recomputed)
  long long mpt;
  if (mid == e.tk_px && mid > 0.0) mpt = e.tk_ticks;
  else { const int t = to_ticks(mk..., mid, &e.err, &e.tk_band); mpt = t; e.tk_px = mid; e.tk_ticks = t; }
  double mpm = mid - m_last_midprice(e), sp = m_spread(e);
  pushv[W_MID] = (double)mpt;
  pushv[W_VLT] = (double)mpt;
  pushv[W_VNUM] = e.side[0].obs_value + e.side[1].obs_value;
  pushv[W_VDEN] = (double)(e.side[0].obs_volume + e.side[1].obs_volume);
  pushv[W_SPREAD] = fmax(0.0, sp);
  pushv[W_TP] = P.tp_is_micro ? m_microprice(e) : mid;  // tp::MicroPrice / tp::MidPrice (target_price.cpp:38-64)
  pushv[W_ASKTX] = (double)e.side[0].obs_volume;
  pushv[W_BIDTX] = (double)e.side[1].obs_volume;
  // EWMA<double>::push (accumulators.cpp:156-163)
  e.ewma_up = (P.ewma_alpha * fmax(0.0, mpm)) + ((1 - P.ewma_alpha) * e.ewma_up);
  e.ewma_dn = (P.ewma_alpha * fabs(fmin(0.0, mpm))) + ((1 - P.ewma_alpha) * e.ewma_dn);
  e.n_ticks++;
}

// BookUtils::IsValidState (book.cpp:612-625); the reference would swallow further rows
__device__ __forceinline__ void check_valid_state(EnvHdr& e) {
  if (e.side[0].has_last && e.side[1].has_last && !(pkey(e.side[0].last_px[0]) == 0.0) && !(pkey(e.side[1].last_px[0]) == 0.0)) {
    double mp = m_midprice(e);
    bool ok = (m_spread(e) >= 0.0) && (mp > 0.0) && (fabs(mp - m_last_midprice(e)) < mp);
    if (!ok) e.err |= ERR_INVALID_STATE;
  }
}

// Intraday::NextState (intraday.cpp:224-272) up to the window pushes, one thread.
template <class... M>
__device__ __noinline__ void next_state_scalar(EnvHdr& e, const rlm_tick_msg& m, double* pushv, M... mk) {
  double mp = m_midprice(e);
  Fill au = side_apply_transactions<true>(e.side[0], m, mp, true);
  Fill bu = side_apply_transactions<false>(e.side[1], m, mp, true);
  update_book_profiles(e, m);
  next_state_tail(e, au, bu, pushv, mk...);
}

// The same with the two book sides on two lanes (they are independent until adverse selection):
// lane 0 = ask, lane 1 = bid.  `fills` = 2 Fill structs + 2 ints of this warp's shared memory.
template <class... M>
__device__ __noinline__ void next_state_warp(EnvHdr& e, const rlm_tick_msg& m, double* pushv, Fill* fills, int lane, M... mk) {
  int* serr = (int*)(fills + 2);
  if (lane < 2) {
    const double mp = m_midprice(e);  // pre-update midprice (intraday.cpp:235)
    serr[lane] = 0;
    fills[lane] = (lane == 0) ? side_apply_transactions<true>(e.side[0], m, mp, true)
                              : side_apply_transactions<false>(e.side[1], m, mp, true);
  }
  __syncwarp();
  if (lane < 2) side_apply_changes(e.side[lane], lane == 0 ? m.ask_px : m.bid_px, lane == 0 ? m.ask_vol : m.bid_vol, m, &serr[lane]);
  __syncwarp();
  if (lane == 0) {
    e.last_date = e.date; e.date = m.date; e.time_ms = m.time_ms;  // intraday.cpp:286-288
    e.err |= serr[0] | serr[1];
    check_valid_state(e);
    next_state_tail(e, fills[0], fills[1], pushv, mk...);
  }
}

// ---------------------------------------------------------------- multi-message ticks (ingested real data)
// One tick = [RLM_TICK_TX_MORE messages] + [depth rows flagged RLM_TICK_PARTIAL] + one last depth row (rlm_flow.h).
// needs_multi: this message cannot take the one-row fast path.
__device__ __forceinline__ bool needs_multi(const EnvHdr& e, const rlm_tick_msg& m) { return (m.flags & 3) != 0 || e.tick_open != 0 || e.txn != 0; }
__device__ __forceinline__ void tick_tx_append(EnvHdr& e, const rlm_tick_msg& m) {
  for (int i = 0; i < m.n_tx && i < RLM_N_TX_MAX; ++i) {
    if (e.txn >= RLM_TX_CAP) { e.err |= ERR_BAD_PRICE; break; }
    e.tx_px[e.txn] = m.tx_px[i]; e.tx_vol[e.txn] = m.tx_vol[i]; e.txn++;
  }
}
// Intraday::UpdateBookProfiles (intraday.cpp:274-313) one depth row at a time; returns true when the tick's last row is in
__device__ __noinline__ bool update_book_profiles_multi(EnvHdr& e, const rlm_tick_msg& m, bool with_tx) {
  if (m.flags & RLM_TICK_TX_MORE) { if (with_tx && !e.tick_open) tick_tx_append(e, m); return false; }
  if (!e.tick_open) {
    if (with_tx) tick_tx_append(e, m); else e.txn = 0;
    side_stash(e.side[0]);
    side_stash(e.side[1]);
  }
  e.last_date = e.date;  // intraday.cpp:286-288, once per row
  e.date = m.date;
  e.time_ms = m.time_ms;
  side_apply_row(e.side[0], m.ask_px, m.ask_vol, e.tx_px, e.tx_vol, e.txn, &e.err);
  side_apply_row(e.side[1], m.bid_px, m.bid_vol, e.tx_px, e.tx_vol, e.txn, &e.err);
  if (m.flags & RLM_TICK_PARTIAL) { e.tick_open = 1; return false; }
  e.tick_open = 0;
  e.txn = 0;
  return true;
}
// Intraday::NextState (intraday.cpp:224-272) for such a tick, one message at a time, one thread; returns true (and fills
// pushv) when the tick is complete
template <class... M>
__device__ __noinline__ bool next_state_multi(EnvHdr& e, const rlm_tick_msg& m, double* pushv, M... mk) {
  if (m.flags & RLM_TICK_TX_MORE) { if (!e.tick_open) tick_tx_append(e, m); return false; }
  if (!e.tick_open) {  // first depth row of the tick: the prints meet the book of the previous tick (intraday.cpp:235-237)
    tick_tx_append(e, m);
    const double mp = m_midprice(e);
    const Fill au = side_apply_transactions_n<true>(e.side[0], e.tx_px, e.tx_vol, e.txn, mp);
    const Fill bu = side_apply_transactions_n<false>(e.side[1], e.tx_px, e.tx_vol, e.txn, mp);
    e.tick_au.volume = au.volume; e.tick_au.proxy = au.proxy; e.tick_au.value = au.value;
    e.tick_bu.volume = bu.volume; e.tick_bu.proxy = bu.proxy; e.tick_bu.value = bu.value;
    side_stash(e.side[0]);
    side_stash(e.side[1]);
  }
  e.last_date = e.date;
  e.date = m.date;
  e.time_ms = m.time_ms;
  side_apply_row(e.side[0], m.ask_px, m.ask_vol, e.tx_px, e.tx_vol, e.txn, &e.err);
  side_apply_row(e.side[1], m.bid_px, m.bid_vol, e.tx_px, e.tx_vol, e.txn, &e.err);
  if (m.flags & RLM_TICK_PARTIAL) { e.tick_open = 1; return false; }
  e.tick_open = 0;
  e.txn = 0;
  check_valid_state(e);
  Fill au, bu;
  au.volume = e.tick_au.volume; au.proxy = e.tick_au.proxy; au.value = e.tick_au.value;
  bu.volume = e.tick_bu.volume; bu.proxy = e.tick_bu.proxy; bu.value = e.tick_bu.value;
  next_state_tail(e, au, bu, pushv, mk...);
  return true;
}

// ulb() of include/utilities/maths.h:4-8 = std::max(std::min(val, ub), lb): a NaN `val` comes back as NaN (both
// comparisons are false), whereas fmin/fmax would drop it -- the vwap variable with an empty volume window is 0/0
__device__ __forceinline__ double ulb_ref(double val, double lb, double ub) {
  const double m = (ub < val) ? ub : val;
  return (m < lb) ? lb : m;
}

// The state variables that convert two prices to ticks (spd, mpm, a_dist, b_dist), split so that the lanes of the
// warp-per-env tick kernel run their Market::ToTicks calls together instead of one switch case after the other.
// var_tick_args: the two prices (returns false for every other variable, and for a dist variable without a live order);
// var_from_ticks: the variable from the two tick counts -- the same expressions as in get_variable below.
__device__ __forceinline__ bool var_tick_args(const EnvHdr& e, const double* ring, int v, double& x0, double& x1) {
  switch (v) {
    case RLM_VAR_SPD: x0 = e.side[0].px[0]; x1 = e.side[1].px[0]; return true;
    case RLM_VAR_MPM: x0 = win_front(e, ring, W_MID); x1 = win_back(e, ring, W_MID); return true;
    case RLM_VAR_A_DIST: if (!e.side[0].ord.live) return false; x0 = e.side[0].ord.price; x1 = e.side[0].px[0]; return true;
    case RLM_VAR_B_DIST: if (!e.side[1].ord.live) return false; x0 = e.side[1].px[0]; x1 = e.side[1].ord.price; return true;
  }
  return false;
}
__device__ __forceinline__ double var_from_ticks(int v, int t0, int t1) {
  switch (v) {
    case RLM_VAR_SPD: return ulb_ref((double)(t0 - t1), 0.0, 20.0);
    case RLM_VAR_MPM: return ulb_ref((double)(t0 - t1), -10.0, 10.0);
  }
  return (double)t0 - (double)t1;  // a_dist / b_dist
}

// Intraday::getVariable (intraday.cpp:315-409)
template <class... M>
__device__ __noinline__ double get_variable(EnvHdr& e, const double* ring, int v, M... mk) {
  switch (v) {
    case RLM_VAR_POS: return (double)e.position / (double)P.order_size;
    case RLM_VAR_SPD: {
      double d = (double)(to_ticks(mk..., e.side[0].px[0], &e.err, &e.tk_band) - to_ticks(mk..., e.side[1].px[0], &e.err, &e.tk_band));
      return ulb_ref(d, 0.0, 20.0);
    }
    case RLM_VAR_MPM: {
      double d = (double)(to_ticks(mk..., win_front(e, ring, W_MID), &e.err, &e.tk_band) - to_ticks(mk..., win_back(e, ring, W_MID), &e.err, &e.tk_band));
      return ulb_ref(d, -10.0, 10.0);
    }
    case RLM_VAR_IMB: {
      double v_a = (double)e.side[0].total_vol, v_b = (double)e.side[1].total_vol;
      return ((v_a + v_b) > 0 ? 5.0 * (v_b - v_a) / (v_b + v_a) : 0.0);
    }
    case RLM_VAR_SVL: {
      double q_a = e.w_sum[W_ASKTX], q_b = e.w_sum[W_BIDTX];
      return ((q_a + q_b) > 0 ? 5.0 * (q_b - q_a) / (q_a + q_b) : 0.0);
    }
    case RLM_VAR_VOL: return ulb_ref(5.0 * win_std(e, W_VLT), 0.0, 10.0);
    case RLM_VAR_RSI: {
      double u = e.ewma_up, d = e.ewma_dn;
      return (u + d) != 0.0 ? 5.0 * (u - d) / (u + d) : 0.0;
    }
    case RLM_VAR_VWAP: {
      double d = e.w_sum[W_VNUM] / e.w_sum[W_VDEN];
      return ulb_ref(d / e.w_mean[W_SPREAD], -10.0, 10.0);
    }
    case RLM_VAR_A_DIST:
      if (e.side[0].ord.live) return ((double)to_ticks(mk..., e.side[0].ord.price, &e.err, &e.tk_band) - (double)to_ticks(mk..., e.side[0].px[0], &e.err, &e.tk_band));
      else return -100.0;
    case RLM_VAR_A_QUEUE:
      if (e.side[0].ord.live) {
        float qp = (float)e.side[0].ord.q_head / fmaxf(1.0f, (float)e.side[0].ord.initial_queue);  // order.cpp:130-133
        return 10.0 * (double)(long long)qp;                                                        // book.cpp:351-357
      } else return -1.0;
    case RLM_VAR_B_DIST:
      if (e.side[1].ord.live) return ((double)to_ticks(mk..., e.side[1].px[0], &e.err, &e.tk_band) - (double)to_ticks(mk..., e.side[1].ord.price, &e.err, &e.tk_band));
      else return -100.0;
    case RLM_VAR_B_QUEUE:
      if (e.side[1].ord.live) {
        float qp = (float)e.side[1].ord.q_head / fmaxf(1.0f, (float)e.side[1].ord.initial_queue);
        return 10.0 * (double)(long long)qp;
      } else return -1.0;
    case RLM_VAR_LAST_ACTION: return (double)e.last_action;
  }
  return 0.0;
}
