// lob_oracle.cpp -- CPU restatement of the rl_markets hot path.
// TEST INFRASTRUCTURE ONLY: see lob_oracle.h for who may load this and how it is pinned.
//
// Every function cites the reference file:line it restates (paths relative to
// /root/reference).  The restatement keeps the reference's fp64 operation order
// (built with -ffp-contract=off, like oracle/_ref) so that it can be compared
// BITWISE with the reference's own output.  It is one-env-at-a-time scalar code
// on purpose: it shares no structure with the CUDA implementation.
#include "lob_oracle.h"

#include <algorithm>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "rlm_flow_tables.h"
#include "rlm_rndseq.h"

namespace {

// =====================================================================================
// RNGs.  The reference consumes libstdc++ std::mt19937_64 through
// uniform_real_distribution<double> / uniform_int_distribution<unsigned>
// (src/rl/policy.cpp:13-15,29,71-72; src/rl/agent.cpp:30-31,334) and glibc rand()
// (src/rl/policy.cpp:49; src/rl/agent.cpp:160,255; seeded at src/main.cpp:87).
// Restated here so that each env owns private generator state.
// =====================================================================================
struct MT64 {  // std::mersenne_twister_engine<uint64,64,312,156,31,...> (ISO C++ [rand.predef])
  uint64_t x[312];
  int p;
  void seed(uint64_t s) {
    x[0] = s;
    for (int i = 1; i < 312; ++i) x[i] = 6364136223846793005ull * (x[i - 1] ^ (x[i - 1] >> 62)) + (uint64_t)i;
    p = 312;
  }
  void twist() {
    const uint64_t UM = 0xFFFFFFFF80000000ull, LM = 0x7FFFFFFFull, A = 0xB5026F5AA96619E9ull;
    for (int k = 0; k < 312; ++k) {
      uint64_t y = (x[k] & UM) | (x[(k + 1) % 312] & LM);
      x[k] = x[(k + 156) % 312] ^ (y >> 1) ^ ((y & 1) ? A : 0);
    }
    p = 0;
  }
  uint64_t next() {
    if (p >= 312) twist();
    uint64_t z = x[p++];
    z ^= (z >> 29) & 0x5555555555555555ull;
    z ^= (z << 17) & 0x71D67FFFEDA60000ull;
    z ^= (z << 37) & 0xFFF7EEE000000000ull;
    z ^= z >> 43;
    return z;
  }
};

// libstdc++ generate_canonical<double,53>(mt19937_64): one draw, double(u)/2^64, clamp below 1
// (/usr/include/c++/13/bits/random.tcc:3349-3381); uniform_real_distribution(0,1) = ret*(1-0)+0.
double uniform_real01(MT64& g) {
  double sum = (double)g.next();
  double ret = sum / 18446744073709551616.0;
  if (ret >= 1.0) ret = std::nextafter(1.0, 0.0);
  return ret * (1.0 - 0.0) + 0.0;
}

// libstdc++ uniform_int_distribution<unsigned>(0,n-1) on a full 64-bit URBG: Lemire's method
// with a 128-bit product (/usr/include/c++/13/bits/uniform_int_dist.h:_S_nd and operator()).
uint32_t uniform_int_n(MT64& g, uint32_t n) {
  uint64_t range = n;
  unsigned __int128 product = (unsigned __int128)g.next() * range;
  uint64_t low = (uint64_t)product;
  if (low < range) {
    uint64_t threshold = (0 - range) % range;
    while (low < threshold) {
      product = (unsigned __int128)g.next() * range;
      low = (uint64_t)product;
    }
  }
  return (uint32_t)(product >> 64);
}

// glibc random_r TYPE_3 (degree 31, separation 3), as used by rand()/srand().
struct GlibcRand {
  int32_t r[31];
  int f, b;
  void seed(uint32_t s) {
    if (s == 0) s = 1;
    r[0] = (int32_t)s;
    for (int i = 1; i < 31; ++i) {
      long hi = r[i - 1] / 127773, lo = r[i - 1] % 127773;
      long word = 16807 * lo - 2836 * hi;
      if (word < 0) word += 2147483647;
      r[i] = (int32_t)word;
    }
    f = 3;
    b = 0;
    for (int i = 0; i < 310; ++i) next();
  }
  int32_t next() {
    uint32_t v = (uint32_t)r[f] + (uint32_t)r[b];
    r[f] = (int32_t)v;
    int32_t out = (int32_t)(v >> 1);
    f = (f + 1) % 31;
    b = (b + 1) % 31;
    return out;
  }
};

// =====================================================================================
// utilities/accumulators  (src/utilities/accumulators.cpp)
// =====================================================================================
struct Accumulator {  // accumulators.cpp:11-76
  size_t window_size = 1;
  std::deque<double> window;
  double sum_ = 0.0;
  void init(size_t w) { window_size = w; window.clear(); sum_ = 0.0; }
  void push(double v) {  // :17-27
    sum_ += v;
    window.push_front(v);
    if (window.size() > window_size) {
      sum_ -= window.back();
      window.pop_back();
    }
  }
  double sum() const { return sum_; }
  double front() const { return window.front(); }
  double back() const { return window.back(); }
  void clear() { window.clear(); }  // :60-64 -- keeps sum_ (SURVEY Appendix A13)
  bool full() const { return window.size() == window_size; }
  size_t size() const { return window.size(); }
};

struct RollingMean : Accumulator {  // accumulators.cpp:80-131
  double mean_ = 0.0, s_ = 0.0;
  void init(size_t w) { Accumulator::init(w); mean_ = 0.0; s_ = 0.0; }
  void push(double val) {  // :86-109
    sum_ += val;
    window.push_front(val);
    double n = (double)window.size();
    double old_mean = mean_;
    mean_ += (val - mean_) / n;
    s_ += (val - mean_) * (val - old_mean);
    if (window.size() > window_size) {
      double old = window.back();
      window.pop_back();
      sum_ -= old;
      double n2 = (double)window.size();
      double old_mean2 = mean_;
      mean_ -= (old - mean_) / n2;
      s_ -= (old - mean_) * (old - old_mean2);
    }
  }
  double mean() const { return mean_; }
  double var() const { return s_ / (double)(window.size() - 1); }  // :117-121 (size_t arithmetic)
  double stddev() const {                                          // :123-131
    double v = var();
    return v > 0 ? std::sqrt(v) : 0.0;
  }
};

struct EWMA {  // accumulators.cpp:148-169; the deque stays empty (push_front + pop_back)
  double alpha = 1.0, mean_ = 0.0;
  void init(size_t w) { alpha = 2.0 / (w + 1.0); mean_ = 0.0; }
  void push(double v) { mean_ = (alpha * v) + ((1 - alpha) * mean_); }
  double mean() const { return mean_; }
  void clear() {}
};

// =====================================================================================
// market/market  (src/market/market.cpp:11-38,67-138)
// =====================================================================================
struct Venue {
  int n = 0;
  double px[RLM_MAX_BANDS], ts[RLM_MAX_BANDS];  // pts_ ascending
  int tts_tick[RLM_MAX_BANDS];                  // tts_ keys (market.cpp:27-37)
  double tts_ts[RLM_MAX_BANDS];
  long mo = 0, mc = 0;
  int date = 0;
  long time = 0;

  void init(const rlm_config* c) {
    n = c->n_bands;
    for (int i = 0; i < n; ++i) { px[i] = c->band_px[i]; ts[i] = c->band_ts[i]; }
    mo = c->open_ms; mc = c->close_ms;
    tts_tick[0] = 0; tts_ts[0] = ts[0];
    long acc_ticks = 0;                                    // market.cpp:30-37
    for (int i = 1; i < n; ++i) {
      acc_ticks += (px[i] - px[i - 1]) / ts[i - 1];        // long += double (truncating)
      tts_tick[i] = (int)acc_ticks;
      tts_ts[i] = ts[i];
    }
    date = 0; time = 0;
  }
  bool IsOpen() const { return (time > mo + 30 * 60000L) && (time < mc - 30 * 60000L); }  // :67-70
  double tick_size(double price) const {  // :130-138 prev(upper_bound(price))
    int k = -1;
    for (int i = 0; i < n; ++i) if (!(price < px[i])) k = i;  // last key <= price
    if (k < 0) throw std::invalid_argument("[Market] Invalid price for tick conversion.");
    return ts[k];
  }
  int ToTicks(double price) const {  // :78-102
    int ticks = 0;
    double ub;
    int it = 0;
    if (price < px[0]) throw std::invalid_argument("[Market] Invalid price for tick conversion.");
    // The reference evaluates the left operand on end() (UB); in practice the stale read is a
    // tiny positive denormal and the right operand ends the loop, i.e. the loop stops after
    // the last band (SURVEY Appendix A16).
    while (it != n && price + tick_size(px[it]) / 2.0 > px[it]) {
      if (it == n - 1 || price < px[it + 1])
        ub = price + tick_size(price) / 2.0;
      else
        ub = px[it + 1];
      ticks += (ub - px[it]) / ts[it];  // int += double (truncating)
      it++;
    }
    return ticks;
  }
  double ToPrice(int ticks) const {  // :104-128
    double price = 0;
    double ub;
    int it = 0;
    if (ticks < tts_tick[0]) throw std::invalid_argument("[Market] Invalid number of ticks for price conversion.");
    while (it != n && ticks > tts_tick[it]) {
      if (it == n - 1 || ticks < tts_tick[it + 1])
        ub = ticks;
      else
        ub = tts_tick[it + 1];
      price += (ub - tts_tick[it]) * tts_ts[it];
      it++;
    }
    return price;
  }
};

// =====================================================================================
// market/order  (src/market/order.cpp)
// =====================================================================================
struct Order {
  bool live = false;
  double price = 0;
  long size = 0, q_head = 0, q_tail = 0, total_executed = 0, initial_queue = 0;
  int transactions = 0;

  void create(double p, long sz, long qh) {  // order.cpp:12-30
    if (p <= 0) throw std::runtime_error("Order price must be non-zero and positive.");
    if (sz <= 0) throw std::runtime_error("Order size must be non-zero and positive.");
    if (qh < 0) throw std::runtime_error("Order queue must be positive.");
    live = true; price = p; size = sz; q_head = qh; q_tail = 0; total_executed = 0; initial_queue = qh;
    transactions = 0;
  }
  long remaining() const { return std::max(size - total_executed, 0L); }  // :34-37
  bool isExecuted() const { return total_executed >= size; }              // :49-52
  long doTransaction(long volume) {                                       // :54-82
    if (volume < 0) throw std::runtime_error("Transaction volume must be positive.");
    transactions += volume;
    long remaining_volume = volume - q_head;
    if (remaining_volume > 0) {
      q_head = 0;
      if (remaining() <= remaining_volume) {
        total_executed = size;
        remaining_volume -= size;
      } else {
        total_executed += remaining_volume;
        remaining_volume = 0;
      }
    } else {
      q_head -= volume;
    }
    return std::max(remaining_volume, 0L);
  }
  void doCancellation(long volume) {  // :84-107
    if (volume < 0) throw std::runtime_error("Cancellation volume must be positive.");
    if (q_tail == 0) {
      q_head -= volume;
    } else {
      double total = q_head + q_tail;
      // `long -= double`: the long is converted to double, the subtraction is done in
      // double and the result converted back (x86: cvttsd2si; inf/NaN -> LONG_MIN).
      q_head = d2l((double)q_head - std::ceil(volume * q_head / total));
      q_tail = d2l((double)q_tail - std::floor(volume * q_tail / total));
    }
    if (q_head < 0) {
      q_tail = (long)((unsigned long)q_tail + (unsigned long)q_head);  // wraps like the x86 add
      q_head = 0;
    }
    if (q_tail < 0) q_tail = 0;
  }
  static long d2l(double d) {
    // x86-64 cvttsd2si semantics for out-of-range / NaN (SURVEY Appendix A5)
    if (!(d > -9.3e18 && d < 9.3e18)) return (long)0x8000000000000000ull;
    return (long)d;
  }
  void addVolumeBehind(long v) { q_tail += v; }  // :109-112
  void clearQueues() { q_head = 0; q_tail = 0; } // :114-118
  float getQueueProgress() const { return q_head / std::max(1.0f, (float)initial_queue); }  // :130-133
};

// =====================================================================================
// market/book  (src/market/book.cpp) -- one agent order per side (ORDER_LIMIT == 1,
// src/environment/base.cpp:21)
// =====================================================================================
inline double pkey(double p) { return std::rint(p * 10000u); }  // utilities/comparison.h:13-16

struct Tx {  // data::TimeAndSalesRecord::transactions (records.h:32), ascending FloatComparator order
  int n = 0;
  double px[RLM_TX_CAP];
  long vol[RLM_TX_CAP];
  long find(double price) const {  // map::find by comparator key
    double k = pkey(price);
    for (int i = 0; i < n; ++i) if (pkey(px[i]) == k) return vol[i];
    return 0L;
  }
};

struct Side {
  bool is_ask = true;
  int depth = RLM_DEPTH;
  double prices[RLM_DEPTH], last_prices[RLM_DEPTH];
  // levels / last_levels: std::map<double,long,C> kept in comparator order
  int n_lv = 0, n_last = 0;
  double lv_px[RLM_DEPTH], last_px[RLM_DEPTH];
  long lv_vol[RLM_DEPTH], last_vol[RLM_DEPTH];
  long total_volume_ = 0, last_total_volume_ = 0;
  int n_transacted_ = 0;
  double observed_value_ = 0.0;
  long observed_volume_ = 0;
  Order o;

  bool before(double a, double b) const {  // comparator (comparison.h:13-29)
    return is_ask ? (pkey(a) < pkey(b)) : (pkey(b) < pkey(a));
  }
  void Reset() {  // book.cpp:143-160
    n_transacted_ = 0; observed_value_ = 0.0; observed_volume_ = 0;
    total_volume_ = 0; last_total_volume_ = 0;
    for (int l = 0; l < RLM_DEPTH; ++l) { prices[l] = 0.0; last_prices[l] = 0.0; }
    n_lv = 0; n_last = 0;
    o.live = false;
  }
  void StashState() {  // :50-55 (swap)
    for (int l = 0; l < RLM_DEPTH; ++l) std::swap(prices[l], last_prices[l]);
    std::swap(n_lv, n_last);
    for (int l = 0; l < RLM_DEPTH; ++l) { std::swap(lv_px[l], last_px[l]); std::swap(lv_vol[l], last_vol[l]); }
  }
  bool HasStash() const { return !(pkey(last_prices[0]) == pkey(0.0)); }  // :57-61
  void level_insert(double p, long v) {  // levels[p] = v
    for (int i = 0; i < n_lv; ++i)
      if (pkey(lv_px[i]) == pkey(p)) { lv_vol[i] = v; return; }
    int pos = n_lv;
    while (pos > 0 && before(p, lv_px[pos - 1])) { lv_px[pos] = lv_px[pos - 1]; lv_vol[pos] = lv_vol[pos - 1]; --pos; }
    lv_px[pos] = p; lv_vol[pos] = v; ++n_lv;
  }
  long volume(double p) const {  // :208-214
    for (int i = 0; i < n_lv; ++i) if (pkey(lv_px[i]) == pkey(p)) return lv_vol[i];
    return 0L;
  }
  long last_volume(double p) const {  // :216-222
    for (int i = 0; i < n_last; ++i) if (pkey(last_px[i]) == pkey(p)) return last_vol[i];
    return 0L;
  }
  double price(int level) const {  // :166-176
    if (level < 0) level = depth + level;
    if (level >= depth || level < 0 || prices[level] == 0.0)
      throw std::runtime_error("Attempted to access an undefined price at level");
    return prices[level];
  }
  double last_price(int level) const {  // :178-188
    if (level < 0) level = depth + level;
    if (level >= depth || level < 0 || last_prices[level] == 0.0)
      throw std::runtime_error("Attempted to access undefined last price at level");
    return last_prices[level];
  }
  void UpdateOrder(long transaction_volume) {  // :101-141
    if (!o.live) return;
    double price = o.price;
    if (o.isExecuted()) { o.live = false; return; }
    long lv = last_volume(price);
    if (lv == 0) return;
    long v = volume(price);
    if (v == 0) { o.clearQueues(); return; }
    long vol_diff = lv - v;
    if (vol_diff >= 0) {
      long cancelled_volume = vol_diff - transaction_volume;
      if (cancelled_volume > 0) o.doCancellation(cancelled_volume);
    } else
      o.addVolumeBehind(vol_diff);
  }
  void ApplyChanges(const double* new_prices, const long* new_volumes, const Tx& tx) {  // :63-99
    n_lv = 0;
    last_total_volume_ = total_volume_;
    for (int l = 0; l < depth; ++l) {
      if (new_prices[l] <= 0.0) throw std::runtime_error("Prices must be non-zero positive");
      else if (new_volumes[l] <= 0) throw std::runtime_error("Volumes must be non-zero positive");
      else {
        prices[l] = new_prices[l];
        level_insert(new_prices[l], new_volumes[l]);
        total_volume_ += new_volumes[l];
      }
    }
    // std::sort(prices, comparator): insertion sort (distinct keys => same result)
    for (int i = 1; i < depth; ++i) {
      double p = prices[i];
      int j = i;
      while (j > 0 && before(p, prices[j - 1])) { prices[j] = prices[j - 1]; --j; }
      prices[j] = p;
    }
    if (o.live) UpdateOrder(tx.find(o.price));
  }
  bool PlaceOrder(double p, long size) {  // :249-261
    if (o.live && pkey(o.price) == pkey(p)) return false;
    o.create(p, size, volume(p));
    return true;
  }
  int order_count() const { return o.live ? 1 : 0; }
  void CancelAll() { o.live = false; }

  // AskBook::ApplyTransactions book.cpp:382-427 / BidBook::ApplyTransactions :467-510
  void ApplyTransactions(const Tx& tx, double ref, long& volume, double& proxy, double& value) {
    observed_value_ = 0.0;
    observed_volume_ = 0L;
    volume = 0L; proxy = 0.0; value = 0.0;
    for (int k = 0; k < tx.n; ++k) {
      int i = is_ask ? k : tx.n - 1 - k;
      double tp = tx.px[i];
      if (is_ask ? (tp < ref) : (tp > ref)) continue;
      long vol = tx.vol[i];
      observed_value_ += tp * vol;
      observed_volume_ += vol;
      while (o.live && (is_ask ? (o.price <= tp) : (o.price >= tp))) {
        long order_rem = o.remaining();
        vol = o.doTransaction(vol);
        long order_exec = order_rem - o.remaining();
        if (is_ask) {
          volume -= order_exec;
          proxy += (o.price - ref) * order_exec;
          value += o.price * order_exec;
        } else {
          volume += order_exec;
          proxy += (ref - o.price) * order_exec;
          value -= o.price * order_exec;
        }
        if (o.isExecuted()) { o.live = false; n_transacted_++; }
        if (vol <= 0) break;
      }
    }
  }
  // AskBook::WalkTheBook :429-456 / BidBook::WalkTheBook :512-539
  void WalkTheBook(double ref, long size, long& out_vol, double& proxy, double& value) {
    long abs_size = std::labs(size);
    out_vol = 0; proxy = 0.0; value = 0.0;
    if (abs_size > total_volume_) return;
    long executed = 0L;
    for (int i = 0; i < n_lv; ++i) {
      long lvol = lv_vol[i], l_ex = std::min(lvol, (abs_size - executed));
      executed += l_ex;
      proxy -= l_ex * std::fabs(lv_px[i] - ref);
      if (is_ask) value -= l_ex * lv_px[i]; else value += l_ex * lv_px[i];
      if (executed >= abs_size) { n_transacted_++; break; }
    }
    out_vol = is_ask ? executed : -executed;
  }
};

// include/market/measures.h
inline double m_spread(const Side& a, const Side& b) { return a.price(0) - b.price(0); }                        // :9-12
inline double m_midprice(const Side& a, const Side& b) { return (a.price(0) + b.price(0)) / 2.0f; }              // :24-27
inline double m_last_midprice(const Side& a, const Side& b) { return (a.last_price(0) + b.last_price(0)) / 2.0f; }  // :29-32
inline double m_midprice_move(const Side& a, const Side& b) { return m_midprice(a, b) - m_last_midprice(a, b); } // :34-37
inline double m_microprice(const Side& a, const Side& b) {                                                       // :39-53
  double ap = a.price(0), bp = b.price(0);
  long av = a.total_volume_, bv = b.total_volume_;
  double div = (double)(av + bv);
  double mpm_a = av * bp;
  double mpm_b = ap * bv;
  return (mpm_a + mpm_b) / div;
}

// BookUtils::HandleAdverseSelection book.cpp:550-592
void adverse_selection(Side& ask, Side& bid, long& volume, double& proxy, double& value) {
  const double bap = ask.price(0), bbp = bid.price(0), rp = m_last_midprice(ask, bid);
  volume = 0L; proxy = 0.0; value = 0.0;
  if (ask.o.live && ask.o.price <= bbp) {
    long rem = ask.o.remaining();
    volume -= rem;
    proxy += rem * (ask.o.price - rp);
    value += rem * ask.o.price;
    ask.o.doTransaction(rem);
    ask.o.live = false;
    ask.n_transacted_++;
  }
  if (bid.o.live && bid.o.price >= bap) {
    long rem = bid.o.remaining();
    volume += rem;
    proxy += rem * (rp - bid.o.price);
    value -= rem * bid.o.price;
    bid.o.doTransaction(rem);
    bid.o.live = false;
    bid.n_transacted_++;
  }
}

// BookUtils::IsValidState book.cpp:612-625
bool is_valid_state(const Side& ask, const Side& bid) {
  double mp = m_midprice(ask, bid);
  if (ask.HasStash() && bid.HasStash())
    return (m_spread(ask, bid) >= 0.0) && (mp > 0.0) && (std::fabs(m_midprice_move(ask, bid)) < mp);
  return true;
}

// =====================================================================================
// rl/tiles  (src/rl/tiles.cpp:31-75 tiles(), :130-169 hash_UNH)
// =====================================================================================
int hash_UNH(const int* ints, int num_ints, long m, int increment) {
  long index;
  long sum = 0;
  for (int i = 0; i < num_ints; i++) {
    index = ints[i];
    index += (increment * i);
    index = index & 2047;
    while (index < 0) index += 2048;
    sum += (long)rlm_rndseq_table[(int)index];
  }
  index = (int)(sum % m);
  while (index < 0) index += m;
  return (int)index;
}

void tiles_one_int(int* the_tiles, int num_tilings, int memory_size, const float* floats, int num_floats, int h1) {
  int qstate[20], base[20], coordinates[20 * 2 + 1];
  int num_coordinates = num_floats + 1 + 1;
  coordinates[num_floats + 1] = h1;
  for (int i = 0; i < num_floats; i++) {
    qstate[i] = (int)std::floor(floats[i] * num_tilings);  // float * int -> float, floor(float) -> float
    base[i] = 0;
  }
  for (int j = 0; j < num_tilings; j++) {
    int i;
    for (i = 0; i < num_floats; i++) {
      if (qstate[i] >= base[i])
        coordinates[i] = qstate[i] - ((qstate[i] - base[i]) % num_tilings);
      else
        coordinates[i] = qstate[i] + 1 + ((base[i] - qstate[i] - 1) % num_tilings) - num_tilings;
      base[i] += 1 + (2 * i);
    }
    coordinates[i] = j;
    the_tiles[j] = hash_UNH(coordinates, num_coordinates, memory_size, 449);
  }
}

// rl/state  (src/rl/state.cpp)
struct State {
  int T = 32, A = 9;
  long M = 0;
  std::vector<float> vars;
  std::vector<std::vector<int>> features;  // [A][3T], zero-initialised (state.cpp:16)
  void init(long m, int a, int t) { M = m; A = a; T = t; vars.clear(); features.assign(a, std::vector<int>(3 * t, 0)); }
  void populate() {  // state.cpp:53-65
    for (int a = 0; a < A; a++) {
      tiles_one_int(&features[a][0], T, (int)M, &vars[0], 3, a);
      tiles_one_int(&features[a][T], T, (int)M, &vars[3], (int)vars.size() - 3, A + a);
      tiles_one_int(&features[a][2 * T], T, (int)M, &vars[0], (int)vars.size(), (2 * A) + a);
    }
  }
};

// rl/traces  (src/rl/traces.cpp)
struct Traces {
  long M = 0; int T = 32, A = 9;
  float tolerance = 0.01f;
  std::vector<float> eligibility;
  std::vector<int> inverse;
  std::vector<int> nonzero;
  int n = 0;
  static const int MAXNZ = 100000;  // traces.h:10
  void init(long m, int t, int a) { M = m; T = t; A = a; tolerance = 0.01; eligibility.assign(m, 0.0f); inverse.assign(m, 0); nonzero.assign(MAXNZ, 0); n = 0; }
  void clearExisting(int f, int loc) {  // :86-92
    eligibility[f] = 0.0;
    n--;
    nonzero[loc] = nonzero[n];
    inverse[nonzero[loc]] = loc;
  }
  void decay(float rate) {  // :30-38
    for (int loc = n - 1; loc >= 0; loc--) {
      int f = nonzero[loc];
      eligibility[f] *= rate;
      if (eligibility[f] < tolerance) clearExisting(f, loc);
    }
  }
  void increaseTolerance() {  // :94-101
    tolerance *= 1.1;
    for (int loc = n - 1; loc >= 0; loc--) {
      int f = nonzero[loc];
      if (eligibility[f] < tolerance) clearExisting(f, loc);
    }
  }
  void set(int f, float value) {  // :67-78
    if (eligibility[f] >= tolerance) eligibility[f] = value;
    else {
      while (n >= MAXNZ) increaseTolerance();
      eligibility[f] = value;
      nonzero[n] = f;
      inverse[f] = n;
      n++;
    }
  }
  void clear(int f) {  // :80-84
    if (eligibility[f] != 0.0) clearExisting(f, inverse[f]);
  }
  void update(State& s, int action) {  // :40-50 -- only the first T features of each action
    for (int a = 0; a < A; a++) {
      std::vector<int> features = s.features[a];
      if (a != action)
        for (int t = 0; t < T; t++) clear(features[t]);
      else
        for (int t = 0; t < T; t++) set(features[t], 1.0);
    }
  }
};

// =====================================================================================
// environment (src/environment/base.cpp, intraday.cpp, risk_manager.cpp) + rl/agent + policy
// =====================================================================================
enum Phase { PH_PREOPEN = 0, PH_WARMUP = 1, PH_RUN = 2, PH_DONE = 3 };

}  // namespace

struct lobo_env {
  rlm_config c;
  int64_t env_index;
  Venue market;
  Side ask, bid;
  long position = 0;  // RiskManager::position_
  // Base members (include/environment/base.h:39-96)
  int last_action = 0, lo_vol_step = 0;
  double pnl_step = 0.0, momentum_pnl_step = 0.0;
  double ask_quote = 0.0, bid_quote = 0.0;
  Accumulator f_vwap_numer, f_vwap_denom;
  RollingMean f_midprice, f_volatility, f_ask_transactions, f_bid_transactions, spread_window, pnl_ups, pnl_downs;
  EWMA return_ups, return_downs;
  RollingMean tp_window;  // tp::MidPrice::mp_ / tp::MicroPrice::mp_
  double tp_val = -1.0;
  bool tp_is_micro = true;
  struct { double reward = 0, pnl = 0, bandh = 0; } episode_stats, experiment_stats;
  struct { int ask_transactions = 0, bid_transactions = 0, market_buys = 0, market_sells = 0; } trade_stats;
  struct { int total_ticks = 0, with_ask = 0, with_bid = 0, with_both = 0, with_pos = 0, t_long = 0, t_short = 0; } tick_stats;
  // Intraday members
  int last_date = 0, ask_level = 0, bid_level = 0;
  // performAction loop state (locals of base.cpp:281-305 kept across ticks)
  double agg_r = 0, agg_pnl = 0, agg_mpm = 0;
  int cur_action = 0;
  // rl
  State state1, state2;
  State *state = nullptr, *last_state = nullptr;
  Traces traces;
  std::vector<double> theta, theta_b;
  // shared-policy batch (SURVEY section 8e): theta lives in the batch object, updates go to dtheta
  std::vector<double>*sh_a = nullptr, *sh_b = nullptr, *sh_da = nullptr, *sh_db = nullptr;
  std::vector<lobo_contrib>* contrib_log = nullptr;  // the batch's contribution log while it is on (lobo_batch_log)
  std::vector<double>& THA() { return sh_a ? *sh_a : theta; }
  std::vector<double>& THB() { return sh_b ? *sh_b : theta_b; }
  bool is_double() const { return c.algorithm == RLM_ALGO_DOUBLE_Q_LEARN || c.algorithm == RLM_ALGO_DOUBLE_R_LEARN; }
  double alpha = 0, eps = 0, eps_init = 0, eps_floor = 0;
  double tau = 0, tau_init = 0, tau_floor = 0;  // Boltzmann (policy.cpp:85-96; read as float, main.cpp:157-158)
  double rho = 0.0;                             // R-learning average reward (agent.h:131,145,157)
  bool greedy = false;
  bool backtest = false;  // Backtester::_step instead of Learner::_step (serial.cpp:121-137)
  MT64 policy_gen, agent_gen;
  GlibcRand crand;
  // bookkeeping
  Phase phase = PH_PREOPEN;
  int64_t total_steps = 0, total_ticks = 0, sum_traces = 0;
  int32_t ep_step = 0;
  double last_reward = 0.0, last_delta = 0.0;
  int invalid_states = 0;

  // ---------------------------------------------------------------------------------
  void init(const rlm_config* cfg, int64_t idx) {
    c = *cfg;
    env_index = idx;
    market.init(cfg);
    ask.is_ask = true; bid.is_ask = false;
    // base.cpp:35-50 (max(lookback,1))
    f_vwap_numer.init(std::max(c.lb_vwap, 1)); f_vwap_denom.init(std::max(c.lb_vwap, 1));
    f_midprice.init(std::max(c.lb_mpm, 1)); f_volatility.init(std::max(c.lb_vlt, 1));
    f_ask_transactions.init(std::max(c.lb_svl, 1)); f_bid_transactions.init(std::max(c.lb_svl, 1));
    spread_window.init(std::max(c.spread_lookback, 1));
    pnl_ups.init(std::max(c.pnl_lookback, 1)); pnl_downs.init(std::max(c.pnl_lookback, 1));
    return_ups.init(std::max(c.lb_rsi, 1)); return_downs.init(std::max(c.lb_rsi, 1));
    // base.cpp:101-112 (inverted selector, SURVEY Appendix A1)
    tp_is_micro = (c.target_price_type == RLM_TP_YAML_MIDPRICE);
    tp_window.init(c.tp_lookback);
    tp_val = -1.0;
    // agent.cpp:14-50
    uint32_t seed = c.random_seed + (uint32_t)idx;
    if (!sh_a) theta.assign(c.memory_size, 0.0);
    bool dbl = (c.algorithm == RLM_ALGO_DOUBLE_Q_LEARN || c.algorithm == RLM_ALGO_DOUBLE_R_LEARN);
    agent_gen.seed(seed);
    if (c.random_init) for (auto& t : theta) t = 2.0 * uniform_real01(agent_gen) - 1.0;  // agent.cpp:37-39
    if (dbl && !sh_b) {
      theta_b.assign(c.memory_size, 0.0);
      if (c.random_init) for (auto& t : theta_b) t = 2.0 * uniform_real01(agent_gen) - 1.0;  // :190-192
    }
    traces.init(c.memory_size, c.n_tilings, c.n_actions);
    alpha = c.alpha_start;
    policy_gen.seed(seed);       // policy.cpp:13
    crand.seed(seed);            // main.cpp:87
    eps_init = (double)c.eps_init; eps = eps_init; eps_floor = (double)c.eps_floor;  // main.cpp:149-154
    tau_init = (double)c.tau_init; tau = tau_init; tau_floor = (double)c.tau_floor;  // main.cpp:157-162
    rho = 0.0;
    state1.init(c.memory_size, c.n_actions, c.n_tilings);
    state2.init(c.memory_size, c.n_actions, c.n_tilings);
    state = &state1; last_state = &state2;  // serial.cpp:14-15
    reset_episode();
  }

  // `environment::Intraday<> env(c)` of main.cpp:219: a NEW env object (window sums, statistics, target price,
  // position all start from scratch) driven by the SAME agent (theta, traces, generators, schedules)
  void new_env() {
    lobo_env* f = new lobo_env();
    f->sh_a = sh_a; f->sh_b = sh_b; f->sh_da = sh_da; f->sh_db = sh_db; f->contrib_log = contrib_log;
    f->init(&c, env_index);
    f->theta.swap(theta); f->theta_b.swap(theta_b);
    f->traces = traces;
    f->policy_gen = policy_gen; f->agent_gen = agent_gen; f->crand = crand;
    f->alpha = alpha; f->eps = eps; f->tau = tau; f->rho = rho; f->greedy = greedy; f->backtest = backtest;
    f->total_steps = total_steps; f->total_ticks = total_ticks; f->sum_traces = sum_traces;
    *this = *f;
    state = &state1; last_state = &state2;
    delete f;
  }

  // Base::Initialise base.cpp:123-135 + Intraday::Initialise intraday.cpp:105-109
  void reset_episode() {
    ask_quote = 0.0; bid_quote = 0.0;
    ask.Reset(); bid.Reset();
    episode_stats = {}; trade_stats = {}; tick_stats = {};
    spread_window.clear(); tp_window.clear();
    f_midprice.clear(); f_volatility.clear(); f_vwap_numer.clear(); f_vwap_denom.clear();
    pnl_ups.clear(); pnl_downs.clear(); f_ask_transactions.clear(); f_bid_transactions.clear();
    last_date = 0; market.date = 0; market.time = 0;
    phase = PH_PREOPEN;
    ep_step = 0;
  }

  // RiskManager risk_manager.cpp:26-39
  void CheckOrders() {
    if (position >= c.pos_ub) bid.CancelAll();
    else if (position <= c.pos_lb) ask.CancelAll();
  }
  void rm_update(long executed) { position += executed; CheckOrders(); }
  // RiskManager::PlaceOrder risk_manager.cpp:61-99 with ORDER_LIMIT 1, auto_cancel
  void rm_place(Side& book, double price, long size) {
    if (book.order_count() < 1) { book.PlaceOrder(price, size); return; }
    book.CancelAll();  // CancelWorst of the only order
    book.PlaceOrder(price, size);
  }

  // Base::getReward base.cpp:166-237
  double getReward() {
    double r = 0.0;
    int abs_pos = std::abs((int)position);
    switch (c.reward_measure) {
      case RLM_REWARD_NONE: break;
      case RLM_REWARD_PNL: r = pnl_step; break;
      case RLM_REWARD_PNL_DAMPED: r = pnl_step - c.damping_factor * std::max(0.0, momentum_pnl_step); break;
      case RLM_REWARD_SPREAD: r = pnl_step / spread_window.mean(); break;
      case RLM_REWARD_NORMED:
        if (!(pnl_ups.full() && pnl_downs.full())) r = 0.0;
        else {
          double u = pnl_ups.mean(), d = pnl_downs.mean();
          double su = pnl_ups.stddev(), sd = pnl_downs.stddev();
          double numer = (u * sd - d * su), denom = (su + sd);
          if (std::isnan(numer) || std::isinf(numer)) numer = 0.0;
          if (std::isnan(denom) || std::isinf(denom)) denom = 0.0;
          r = (std::fabs(denom) < 1e-5) ? numer : (numer / denom);
        }
        break;
      case RLM_REWARD_LOVOL: r = lo_vol_step; break;
      case RLM_REWARD_MM_LINEAR: r = -c.pos_weight * abs_pos; r += c.pnl_weight * pnl_step; break;
      case RLM_REWARD_MM_EXP: r = -std::pow(1.0 - std::exp(c.pos_weight * abs_pos), 2); r += c.pnl_weight * pnl_step; break;
      case RLM_REWARD_MM_DIV:
        if (pnl_step > 0) r = pnl_step / std::max(1.0, (double)abs_pos);
        else r = pnl_step;
    }
    return r * 100;
  }

  // Base::ClearInventory base.cpp:339-349 + RiskManager::ClearInventory/MarketOrder :101-113
  // + BookUtils::MarketOrder book.cpp:594-610
  void ClearInventory() {
    long size = -position;
    long v = 0; double proxy = 0.0, value = 0.0;
    double mip = m_midprice(ask, bid);
    if (size == 0L) { v = 0; proxy = 0.0; value = 0.0; }
    else if (size > 0) ask.WalkTheBook(mip, size, v, proxy, value);
    else bid.WalkTheBook(mip, size, v, proxy, value);
    position += v;
    pnl_step += proxy;
    lo_vol_step += std::labs(v);
    episode_stats.pnl += value;
    if (v > 0) trade_stats.market_buys++;
    else if (v < 0) trade_stats.market_sells++;
  }

  // Intraday l2p_ + _place_orders intraday.cpp:64-82,163-173
  void place_orders(int al, int bl) {
    ask_level = al; bid_level = bl;
    if (c.target_price_type == RLM_TP_YAML_BOOK) {
      ask_quote = market.ToPrice(market.ToTicks(ask.price(0)) + al);
      bid_quote = market.ToPrice(market.ToTicks(bid.price(0)) - bl);
    } else {
      double tp = tp_val, half_spd = std::max(0.0, spread_window.mean() / 2.0);
      ask_quote = market.ToPrice(market.ToTicks(tp + al * half_spd));
      bid_quote = market.ToPrice(market.ToTicks(tp - bl * half_spd));
    }
    rm_place(ask, ask_quote, c.order_size);
    rm_place(bid, bid_quote, c.order_size);
  }

  // Intraday::DoAction intraday.cpp:175-220
  void DoAction(int action) {
    switch (action) {
      case 0: place_orders(1, 1); break;
      case 1: ClearInventory(); place_orders(ask_level, bid_level); break;
      case 2: place_orders(2, 2); break;
      case 3: place_orders(3, 3); break;
      case 4: place_orders(0, 2); break;
      case 5: place_orders(2, 0); break;
      case 6: place_orders(1, 4); break;
      case 7: place_orders(4, 1); break;
      case 8: place_orders(5, 5); break;
    }
  }

  // Base::UpdateStats base.cpp:412-442
  void UpdateStats() {
    trade_stats.ask_transactions = ask.n_transacted_;
    trade_stats.bid_transactions = bid.n_transacted_;
    tick_stats.total_ticks++;
    bool has_ask = ask.order_count() > 0, has_bid = bid.order_count() > 0;
    if (has_ask) tick_stats.with_ask++;
    if (has_bid) tick_stats.with_bid++;
    if (has_ask && has_bid) tick_stats.with_both++;
    if (position != 0) tick_stats.with_pos++;
    if (position > 0) tick_stats.t_long++; else if (position < 0) tick_stats.t_short++;
  }

  // One tick of the packed stream = [RLM_TICK_TX_MORE messages] + [depth rows flagged RLM_TICK_PARTIAL] + one last depth
  // row (include/rlm_flow.h).  The synthetic flow has exactly one message per tick.
  struct TickGroup { Tx tx; std::vector<const rlm_tick_msg*> rows; };
  // collects the group that starts at msgs[i]; false (i untouched) if the buffer ends inside it
  static bool take_group(const rlm_tick_msg* msgs, int64_t n, int64_t& i, TickGroup& g) {
    g.tx.n = 0; g.rows.clear();
    int64_t k = i;
    auto add_tx = [&](const rlm_tick_msg& m) {
      for (int t = 0; t < m.n_tx && g.tx.n < RLM_TX_CAP; ++t) { g.tx.px[g.tx.n] = (double)m.tx_px[t]; g.tx.vol[g.tx.n] = m.tx_vol[t]; g.tx.n++; }
    };
    while (k < n && (msgs[k].flags & RLM_TICK_TX_MORE)) add_tx(msgs[k++]);
    bool first = true;
    while (k < n) {
      const rlm_tick_msg& m = msgs[k++];
      if (first) { add_tx(m); first = false; }
      g.rows.push_back(&m);
      if (!(m.flags & RLM_TICK_PARTIAL)) { i = k; return true; }
    }
    return false;
  }

  // Intraday::UpdateBookProfiles intraday.cpp:274-313: one StashState, then every depth row of the tick
  void UpdateBookProfiles(const TickGroup& g, const Tx& tx) {
    ask.StashState(); bid.StashState();
    for (const rlm_tick_msg* pm : g.rows) {
      const rlm_tick_msg& m = *pm;
      last_date = market.date;
      market.date = m.date; market.time = m.time_ms;
      double ap[RLM_DEPTH], bp[RLM_DEPTH]; long av[RLM_DEPTH], bv[RLM_DEPTH];
      for (int l = 0; l < RLM_DEPTH; ++l) { ap[l] = (double)m.ask_px[l]; bp[l] = (double)m.bid_px[l]; av[l] = m.ask_vol[l]; bv[l] = m.bid_vol[l]; }
      ask.ApplyChanges(ap, av, tx);
      bid.ApplyChanges(bp, bv, tx);
    }
    if (!is_valid_state(ask, bid)) invalid_states++;
  }

  bool isTerminal() const {  // intraday.cpp:152-157
    return (!market.IsOpen()) || ((last_date != 0) && (market.date != last_date));
  }

  // Intraday::NextState intraday.cpp:224-272
  void NextState(const TickGroup& g) {
    const Tx& tx = g.tx;
    double mp = m_midprice(ask, bid);
    long au0, bu0; double au1, au2, bu1, bu2;
    ask.ApplyTransactions(tx, mp, au0, au1, au2);
    bid.ApplyTransactions(tx, mp, bu0, bu1, bu2);
    UpdateBookProfiles(g, tx);
    long as0; double as1, as2;
    adverse_selection(ask, bid, as0, as1, as2);
    pnl_step += au1 + bu1 + as1;
    lo_vol_step += bu0 - au0 + std::labs(as0);
    episode_stats.pnl += au2 + bu2 + as2;
    rm_update(bu0 + au0 + as0);
    long mpt = market.ToTicks(m_midprice(ask, bid));
    double mpm = m_midprice_move(ask, bid), sp = m_spread(ask, bid);
    f_midprice.push(mpt);
    f_volatility.push(mpt);
    f_vwap_numer.push(ask.observed_value_ + bid.observed_value_);
    f_vwap_denom.push(ask.observed_volume_ + bid.observed_volume_);
    spread_window.push(std::max(0.0, sp));
    // target_price_->update  (target_price.cpp:38-64)
    tp_window.push(tp_is_micro ? m_microprice(ask, bid) : m_midprice(ask, bid));
    tp_val = tp_window.mean();
    return_ups.push(std::max(0.0, mpm));
    return_downs.push(std::fabs(std::min(0.0, mpm)));
    f_ask_transactions.push(ask.observed_volume_);
    f_bid_transactions.push(bid.observed_volume_);
    total_ticks++;
  }

  // Intraday::getVariable intraday.cpp:315-409
  double getVariable(int v) {
    auto ulb = [](double val, double lb, double ub) { return std::max(std::min(val, ub), lb); };
    switch (v) {
      case RLM_VAR_POS: return double(position) / c.order_size;
      case RLM_VAR_SPD: return ulb((double)(market.ToTicks(ask.price(0)) - market.ToTicks(bid.price(0))), 0.0, 20.0);
      case RLM_VAR_MPM: return ulb((double)(market.ToTicks(f_midprice.front()) - market.ToTicks(f_midprice.back())), -10.0, 10.0);
      case RLM_VAR_IMB: {
        double v_a = (double)ask.total_volume_, v_b = (double)bid.total_volume_;
        return ((v_a + v_b) > 0 ? 5 * (v_b - v_a) / (v_b + v_a) : 0.0);
      }
      case RLM_VAR_SVL: {
        double q_a = (double)f_ask_transactions.sum(), q_b = (double)f_bid_transactions.sum();
        return ((q_a + q_b) > 0 ? 5 * (q_b - q_a) / (q_a + q_b) : 0.0);
      }
      case RLM_VAR_VOL: return ulb(5.0 * f_volatility.stddev(), 0.0, 10.0);
      case RLM_VAR_RSI: {
        double u = return_ups.mean(), d = return_downs.mean();
        return (u + d) != 0.0 ? 5.0 * (u - d) / (u + d) : 0.0;
      }
      case RLM_VAR_VWAP: {
        double d = f_vwap_numer.sum() / f_vwap_denom.sum();
        return ulb(d / spread_window.mean(), -10.0, 10.0);
      }
      case RLM_VAR_A_DIST:
        if (ask.order_count() > 0) return ((double)market.ToTicks(ask.o.price) - (double)market.ToTicks(ask.price(0)));
        else return -100.0;
      case RLM_VAR_A_QUEUE:
        if (ask.order_count() > 0) return 10.0 * (long)ask.o.getQueueProgress();  // book.cpp:351-357 returns long
        else return -1.0;
      case RLM_VAR_B_DIST:
        if (bid.order_count() > 0) return ((double)market.ToTicks(bid.price(0)) - (double)market.ToTicks(bid.o.price));
        else return -100.0;
      case RLM_VAR_B_QUEUE:
        if (bid.order_count() > 0) return 10.0 * (long)bid.o.getQueueProgress();
        else return -1.0;
      case RLM_VAR_LAST_ACTION: return last_action;
      default: throw std::invalid_argument("Unknown state-var enum value");
    }
  }
  void newState(State* s) {  // State::newState state.cpp:35-43 + Intraday::getState :411-416
    s->vars.clear();
    for (int i = 0; i < c.n_state_vars; ++i) s->vars.push_back((float)getVariable(c.state_vars[i]));
    s->populate();
  }

  // ---- agent (src/rl/agent.cpp) ----
  double getQ_tab(const std::vector<double>& th, State& s, int action) {  // :117-135 / :211-230
    std::vector<int> features = s.features[action];
    const int T = c.n_tilings;
    double Q = 0.0;
    double w = c.group_weights[0];
    for (int i = 0; i < T; i++) Q += w * th[features[i]];
    w = c.group_weights[1];
    for (int i = T; i < 2 * T; i++) Q += w * th[features[i]];
    w = c.group_weights[2];
    for (int i = T; i < 3 * T; i++) Q += w * th[features[i]];  // starts at T (SURVEY Appendix A8)
    return Q;
  }
  double getQ(State& s, int a) { return getQ_tab(THA(), s, a); }
  double getQb(State& s, int a) { return getQ_tab(THB(), s, a); }
  int argmax_tab(const std::vector<double>& th, State& s) {  // :144-169 / :239-264
    int index = 0, n_ties = 1;
    double currMaxQ = getQ_tab(th, s, index);
    for (int a = 1; a < c.n_actions; a++) {
      double val = getQ_tab(th, s, a);
      if (val >= currMaxQ) {
        if (val > currMaxQ) { currMaxQ = val; index = a; }
        else {
          n_ties++;
          if (0 == crand.next() % n_ties) { currMaxQ = val; index = a; }
        }
      }
    }
    return index;
  }
  int argmaxQ(State& s) { return argmax_tab(THA(), s); }
  int argmaxQb(State& s) { return argmax_tab(THB(), s); }
  double maxQ(State& s) { return getQ(s, argmaxQ(s)); }  // :171-174
  void updateQ_tab(std::vector<double>& th, double update) {  // :137-142 / :232-237
    double scaled_update = update / c.n_tilings;
    if (contrib_log) {  // shared-policy batch with the log on: the same additions, each one also recorded
      const int32_t table = (&th == sh_db) ? 1 : 0;
      for (int k = 0; k < traces.n; ++k) {
        int f = traces.nonzero[k];
        double v = scaled_update * traces.eligibility[f];
        th[f] += v;
        contrib_log->push_back({table, f, v});
      }
      return;
    }
    for (int k = 0; k < traces.n; ++k) { int f = traces.nonzero[k]; th[f] += scaled_update * traces.eligibility[f]; }
  }
  // policies (src/rl/policy.cpp)
  unsigned greedy_sample(std::vector<double>& qs) {  // :37-55
    int argmax = 0, n_ties = 1;
    for (int a = 1; a < c.n_actions; a++) {
      if (qs[a] > qs[argmax]) argmax = a;
      else if (qs[a] >= qs[argmax]) {
        n_ties++;
        if (0 == crand.next() % n_ties) argmax = a;
      }
    }
    return argmax;
  }
  unsigned policy_sample(std::vector<double>& qs) {
    int pt = greedy ? RLM_POLICY_GREEDY : c.policy_type;
    switch (pt) {
      case RLM_POLICY_GREEDY: return greedy_sample(qs);
      case RLM_POLICY_RANDOM: return uniform_int_n(policy_gen, c.n_actions);  // :27-30
      case RLM_POLICY_EPSILON_GREEDY:                                          // :69-75
        if (uniform_real01(policy_gen) < eps) return uniform_int_n(policy_gen, c.n_actions);
        else return greedy_sample(qs);
      case RLM_POLICY_BOLTZMANN: {  // :98-115 (libm exp: bitwise only against the same libm)
        std::vector<double> probabilities(c.n_actions, 0.0);
        double z = 0.0;
        for (int a = 0; a < c.n_actions; a++) { probabilities[a] = std::exp(qs[a] / tau); z += probabilities[a]; }
        double acc = 0.0;
        double r = uniform_real01(policy_gen);
        for (int a = 0; a < c.n_actions; a++) {
          acc += probabilities[a] / z;
          if (r < acc) return a;
        }
        return c.n_actions - 1;
      }
      default: throw std::runtime_error("oracle: unknown policy");
    }
  }
  unsigned agent_action(State& s) {  // Agent::action :67-74 / DoubleAgent::action :202-209
    std::vector<double> qs(c.n_actions, 0.0);
    bool dbl = is_double();
    for (int a = 0; a < c.n_actions; a++) qs[a] = dbl ? (getQ(s, a) + getQb(s, a)) / 2.0f : getQ(s, a);
    return policy_sample(qs);
  }
  void UpdateTraces(State& from, int action) {
    float gl = (float)(c.gamma * c.lambda);  // decay(float rate)
    if (c.algorithm == RLM_ALGO_SARSA || c.algorithm == RLM_ALGO_ONLINE_R_LEARN) {  // Agent::UpdateTraces :111-115
      traces.decay(gl);
    } else {  // QLearn :272-280, DoubleQLearn :319-327, RLearn, DoubleRLearn
      int amax = argmaxQ(from);
      if (action != amax) traces.decay(0.0f); else traces.decay(gl);
    }
    traces.update(from, action);
  }
  double UpdateWeights(State& from, int action, double reward, State& to) {
    const double gamma = c.gamma;
    const double F_term = gamma * 0.0 - 0.0;  // potentials are 0 (base.cpp:239-242)
    double delta;
    switch (c.algorithm) {
      case RLM_ALGO_Q_LEARN: {  // :282-292
        double Q = getQ(from, action);
        delta = reward + F_term + gamma * maxQ(to) - Q;
        updateQ_tab(sh_da ? *sh_da : theta, alpha * delta);
        return delta;
      }
      case RLM_ALGO_SARSA: {  // :300-311
        double Q1 = getQ(from, action), Q2 = getQ(to, (int)agent_action(to));
        delta = reward + F_term + gamma * Q2 - Q1;
        updateQ_tab(sh_da ? *sh_da : theta, alpha * delta);
        return delta;
      }
      case RLM_ALGO_DOUBLE_Q_LEARN: {  // :329-353
        if (uniform_real01(agent_gen) > 0.5) {
          double Qa = getQ(from, action);
          delta = reward + F_term + gamma * getQb(to, argmaxQ(to)) - Qa;
          updateQ_tab(sh_da ? *sh_da : theta, alpha * delta);
        } else {
          double Qb = getQb(from, action);
          delta = reward + F_term + gamma * getQ(to, argmaxQb(to)) - Qb;
          updateQ_tab(sh_db ? *sh_db : theta_b, alpha * delta);
        }
        return delta;
      }
      case RLM_ALGO_R_LEARN: {  // :373-388
        double Q = getQ(from, action), mQ = maxQ(to);
        delta = reward - rho + mQ - Q;
        double update = alpha * delta;
        updateQ_tab(theta, update);
        double nQ = Q + update;
        if (nQ - maxQ(from) < 1e-7) rho += c.beta * (reward - rho + mQ - nQ);
        return delta;
      }
      case RLM_ALGO_ONLINE_R_LEARN: {  // :398-413
        double Q = getQ(from, action), gQ = getQ(to, (int)agent_action(to));
        delta = reward - rho + gQ - Q;
        double update = alpha * delta;
        updateQ_tab(theta, update);
        double nQ = Q + update;
        if (nQ - maxQ(from) < 1e-7) rho += c.beta * (reward - rho + gQ - nQ);
        return delta;
      }
      case RLM_ALGO_DOUBLE_R_LEARN: {  // :432-467
        double Q, mQ;
        if (uniform_real01(agent_gen) > 0.5) {
          Q = getQ(from, action);
          mQ = getQb(to, argmaxQ(to));
          delta = reward - rho + mQ - Q;
          updateQ_tab(theta, alpha * delta);
        } else {
          Q = getQb(from, action);
          mQ = getQ(to, argmaxQb(to));
          delta = reward - rho + mQ - Q;
          updateQ_tab(theta_b, alpha * delta);
        }
        mQ = -DBL_MAX;
        for (int i = 0; i < c.n_actions; i++) {
          double val = (getQ(from, i) + getQb(from, i)) / 2.0;
          if (val > mQ) mQ = val;
        }
        double nQ = Q + alpha * delta;
        if (nQ - mQ < 1e-7) rho += c.beta * (reward - rho + mQ - nQ);
        return delta;
      }
      default: throw std::runtime_error("oracle: unknown algorithm");
    }
  }
  void HandleTerminal(int episode) {  // agent.cpp:103-109 + policy.cpp:79-82
    traces.decay(0.0f);
    alpha = std::max(c.alpha_floor, c.alpha_start * std::pow(c.omega, (double)episode));
    if (c.policy_type == RLM_POLICY_EPSILON_GREEDY) eps = eps_init * std::pow(eps_floor / eps_init, (double)episode / (long)c.eps_T);
    if (c.policy_type == RLM_POLICY_BOLTZMANN) tau = tau_init * std::pow(tau_floor / tau_init, (double)episode / (long)c.tau_T);  // :119-122
  }

  // ---- the learner loop as a tick-driven state machine ----
  // begin of Learner::_step (serial.cpp:55-61) up to the first NextState of performAction
  // (base.cpp:254-284).  Returns false when the episode is over.
  bool begin_step() {
    if (backtest) {  // Backtester::_step serial.cpp:121-128: no swap, the state is rebuilt from the env
      if (isTerminal()) { finish_episode(); return false; }
      newState(state);
      cur_action = (int)agent_action(*state);
    } else {
      std::swap(state, last_state);
      if (isTerminal()) { finish_episode(); return false; }
      cur_action = (int)agent_action(*last_state);
    }
    last_action = cur_action;
    lo_vol_step = 0;
    pnl_step = 0.0;
    momentum_pnl_step = 0.0;
    DoAction(cur_action);
    CheckOrders();
    UpdateStats();
    agg_r = getReward();
    agg_pnl = pnl_step;
    agg_mpm = 0.0;
    return true;
  }
  void finish_episode() {  // Runner::RunEpisode serial.cpp:31
    ClearInventory();
    phase = PH_DONE;
  }

  // one tick of the do-while of base.cpp:285-305; returns true when the loop exits
  bool run_tick(const TickGroup& m) {
    pnl_step = 0.0;
    NextState(m);
    double mpm = m_midprice_move(ask, bid);
    pnl_step += position * mpm;
    momentum_pnl_step += position * mpm;
    agg_r += getReward();
    agg_pnl += pnl_step;
    agg_mpm += mpm;
    return !(!isTerminal() && std::fabs(agg_mpm) < 1e-5);
  }
  // end of performAction (base.cpp:317-336) + serial.cpp:64-67
  void end_step(rlm_step_record* rec) {
    pnl_step = agg_pnl;
    pnl_ups.push(std::max(0.0, pnl_step));
    pnl_downs.push(std::fabs(std::min(0.0, pnl_step)));
    episode_stats.reward += agg_r; experiment_stats.reward += agg_r;
    experiment_stats.pnl += agg_pnl;
    episode_stats.bandh += agg_mpm; experiment_stats.bandh += agg_mpm;
    if (backtest) {  // no newState / HandleTransition after performAction (serial.cpp:130-136)
      double reward = getReward();
      last_reward = reward; last_delta = 0.0;
      if (rec) fill_record(rec, reward, 0.0);
      total_steps++; ep_step++;
      return;
    }
    newState(state);
    double reward = getReward();
    // Agent::HandleTransition agent.cpp:86-101
    UpdateTraces(*last_state, cur_action);
    double delta = UpdateWeights(*last_state, cur_action, reward, *state);
    last_reward = reward; last_delta = delta;
    sum_traces += traces.n;
    if (rec) fill_record(rec, reward, delta);
    total_steps++; ep_step++;
  }

  void fill_order(const Side& s, rlm_order_rec& o) {
    memset(&o, 0, sizeof(o));
    if (s.o.live) {
      o.exists = 1; o.price = s.o.price; o.q_head = s.o.q_head; o.q_tail = s.o.q_tail;
      o.executed = s.o.size - s.o.remaining();
    }
  }
  void fill_record(rlm_step_record* r, double reward, double delta) {
    memset(r, 0, sizeof(*r));
    r->step = ep_step; r->action = cur_action; r->time_ms = (int32_t)market.time; r->terminal = isTerminal() ? 1 : 0;
    r->position = position; r->ask_quote = ask_quote; r->bid_quote = bid_quote;
    r->ask_level = ask_level; r->bid_level = bid_level;
    r->reward = reward; r->pnl_step = pnl_step;
    r->ep_pnl = episode_stats.pnl; r->ep_reward = episode_stats.reward; r->ep_bandh = episode_stats.bandh;
    r->midprice = m_midprice(ask, bid); r->spread = m_spread(ask, bid); r->bandh_step = agg_mpm;  // intraday.cpp:437-451
    fill_order(ask, r->ask); fill_order(bid, r->bid);
    r->ask_transactions = ask.n_transacted_; r->bid_transactions = bid.n_transacted_;
    r->market_buys = trade_stats.market_buys; r->market_sells = trade_stats.market_sells;
    r->lo_vol_step = lo_vol_step;
    r->n_state = (int32_t)state->vars.size();
    for (size_t i = 0; i < state->vars.size() && i < RLM_N_STATE_MAX; ++i) r->state[i] = state->vars[i];
    r->delta = delta;
    r->n_traces = traces.n;
    uint64_t h = 0;
    for (int k = 0; k < traces.n; ++k) {
      int f = traces.nonzero[k];
      uint32_t eb; uint64_t tb; float e = traces.eligibility[f]; double t = THA()[f];
      memcpy(&eb, &e, 4); memcpy(&tb, &t, 8);
      h += rlm_trace_mix((uint32_t)f, eb, tb);
    }
    r->trace_hash = h;
  }

  bool windows_full() const {  // intraday.cpp:119-126
    return f_ask_transactions.full() && f_bid_transactions.full() && f_vwap_numer.full() && f_vwap_denom.full() &&
           f_volatility.full() && f_midprice.full() && tp_window.full() && spread_window.full();
  }

  // shared-policy batch: one tick; returns true when a learner step ended and begin_step() is pending
  // (it must run only after the batch applied theta += dtheta)
  bool tick_deferred(const rlm_tick_msg& one, rlm_step_record* rec) {
    if (phase == PH_DONE) return false;
    TickGroup m;
    int64_t at = 0;
    if (!take_group(&one, 1, at, m)) throw std::runtime_error("the shared-policy batch takes one-message ticks");
    if (phase == PH_PREOPEN) {
      Tx none;
      UpdateBookProfiles(m, none);
      if (market.IsOpen()) phase = PH_WARMUP;
      return false;
    }
    if (phase == PH_WARMUP) {
      NextState(m);
      if (windows_full()) {
        place_orders(1, 1);
        newState(last_state);
        phase = PH_RUN;
        begin_step();  // Q(null state) under theta_t: nothing to wait for
      }
      return false;
    }
    if (run_tick(m)) { end_step(rec); return true; }
    return false;
  }

  int64_t run(const rlm_tick_msg* msgs, int64_t n_msgs, int64_t max_steps, rlm_step_record* recs, int64_t rec_cap,
              int64_t* n_consumed) {
    int64_t steps = 0, i = 0, nrec = 0;
    TickGroup m;
    while (i < n_msgs && phase != PH_DONE) {
      if (max_steps >= 0 && steps >= max_steps) break;
      if (!take_group(msgs, n_msgs, i, m)) break;  // the buffer ends inside a multi-message tick
      if (phase == PH_PREOPEN) {  // intraday.cpp:111-116
        Tx none;
        UpdateBookProfiles(m, none);
        if (market.IsOpen()) phase = PH_WARMUP;
      } else if (phase == PH_WARMUP) {  // intraday.cpp:118-135 + serial.cpp:24-25
        NextState(m);
        if (windows_full()) {
          place_orders(1, 1);
          newState(last_state);
          phase = PH_RUN;
          begin_step();
        }
      } else {
        if (run_tick(m)) {
          end_step((recs && nrec < rec_cap) ? &recs[nrec] : nullptr);
          if (recs && nrec < rec_cap) nrec++;
          steps++;
          begin_step();
        }
      }
    }
    if (n_consumed) *n_consumed = i;
    return steps;
  }
};

// =====================================================================================
// C ABI
// =====================================================================================
extern "C" {

lobo_env* lobo_create(const rlm_config* cfg, int64_t env_index) {
  try {
    lobo_env* e = new lobo_env();
    e->init(cfg, env_index);
    return e;
  } catch (const std::exception& ex) {
    fprintf(stderr, "lobo_create: %s\n", ex.what());
    return nullptr;
  }
}
void lobo_destroy(lobo_env* e) { delete e; }

int64_t lobo_run(lobo_env* e, const rlm_tick_msg* msgs, int64_t n_msgs, int64_t max_steps, rlm_step_record* recs,
                 int64_t rec_cap, int64_t* n_consumed) {
  try {
    return e->run(msgs, n_msgs, max_steps, recs, rec_cap, n_consumed);
  } catch (const std::exception& ex) {
    fprintf(stderr, "lobo_run: exception: %s\n", ex.what());
    return -1;
  }
}
int lobo_is_terminal(lobo_env* e) { return e->phase == PH_DONE; }
void lobo_stats(lobo_env* e, rlm_env_stats* out) {
  memset(out, 0, sizeof(*out));
  out->episode_reward = e->episode_stats.reward; out->episode_pnl = e->episode_stats.pnl; out->episode_bandh = e->episode_stats.bandh;
  out->position = e->position;
  out->ask_transactions = e->ask.n_transacted_; out->bid_transactions = e->bid.n_transacted_;
  out->market_buys = e->trade_stats.market_buys; out->market_sells = e->trade_stats.market_sells;
  out->total_ticks = e->tick_stats.total_ticks; out->steps = e->ep_step;
  out->terminal = e->phase == PH_DONE; out->phase = e->phase;
}
int64_t lobo_total_steps(lobo_env* e) { return e->total_steps; }
int64_t lobo_total_ticks(lobo_env* e) { return e->total_ticks; }
int64_t lobo_sum_traces(lobo_env* e) { return e->sum_traces; }
const double* lobo_theta(lobo_env* e, int table) { return table == 0 ? e->theta.data() : (e->theta_b.empty() ? nullptr : e->theta_b.data()); }
double lobo_rho(lobo_env* e) { return e->rho; }
void lobo_handle_terminal(lobo_env* e, int episode) { e->HandleTerminal(episode); }
// next episode of the SAME experiment::serial::Learner (src/main.cpp:47-58: one `experiment` object per training thread):
// Intraday::Initialise + rewound data.  The two State objects of Runner (serial.h:17-23) are NOT re-created, so the
// first action of the new episode is chosen from -- and the first transition starts at -- the State that was the
// from-state of the previous episode's last completed transition (serial.cpp:24-25,55,60): kept as is.
void lobo_reset(lobo_env* e) { e->reset_episode(); }
// a FRESH Learner (never-populated States, serial.cpp:9-16) on the same env and agent
void lobo_reset_fresh_learner(lobo_env* e) {
  e->state1.init(e->c.memory_size, e->c.n_actions, e->c.n_tilings);
  e->state2.init(e->c.memory_size, e->c.n_actions, e->c.n_tilings);
  e->state = &e->state1; e->last_state = &e->state2;
  e->reset_episode();
}
void lobo_go_greedy(lobo_env* e) { e->greedy = true; }
void lobo_set_backtest(lobo_env* e, int on) { e->backtest = on != 0; }
void lobo_new_env(lobo_env* e) { e->new_env(); }

int64_t lobo_run_batch(const rlm_config* cfg, int32_t n_envs, int64_t n_ticks, int32_t n_threads, int64_t* total_ticks,
                       double* seconds) {
  std::vector<int64_t> steps(n_threads, 0), ticks(n_threads, 0);
  auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> th;
  for (int t = 0; t < n_threads; ++t) {
    th.emplace_back([&, t]() {
      const int CH = 1024;
      std::vector<rlm_tick_msg> buf(CH);
      for (int b = t; b < n_envs; b += n_threads) {
        lobo_env* e = lobo_create(cfg, cfg->env_index0 + b);
        if (!e) continue;
        rlm_flow_state fs;
        rlm_flow_init(&fs, &cfg->flow, (uint64_t)(cfg->env_index0 + b));
        int64_t done = 0;
        while (done < n_ticks && e->phase != PH_DONE) {
          int n = (int)std::min<int64_t>(CH, n_ticks - done);
          for (int i = 0; i < n; ++i)
            rlm_flow_next(&fs, &cfg->flow, rlm_flow_skellam20_lut, rlm_flow_pois30_lut, rlm_flow_pois1p5_lut, &buf[i]);
          int64_t used = 0;
          int64_t s = e->run(buf.data(), n, -1, nullptr, 0, &used);
          steps[t] += s;
          done += n;
        }
        ticks[t] += e->total_ticks;
        lobo_destroy(e);
      }
    });
  }
  for (auto& x : th) x.join();
  auto t1 = std::chrono::steady_clock::now();
  if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
  int64_t s = 0, k = 0;
  for (int t = 0; t < n_threads; ++t) { s += steps[t]; k += ticks[t]; }
  if (total_ticks) *total_ticks = k;
  return s;
}

// ---- shared-policy batch (the reference analogue is threads sharing one Agent*, src/main.cpp:196-206;
// this synchronous formulation -- all envs of a tick read theta_t, theta_{t+1} = theta_t + sum of their
// updates -- is the new algorithm of SURVEY section 8e, restated here as its CPU oracle)
struct lobo_batch {
  rlm_config c;
  std::vector<lobo_env*> envs;
  std::vector<double> th_a, th_b, d_a, d_b;
  std::vector<int> pending;
  std::vector<lobo_contrib> log;  // this tick's dtheta additions, in the order they were made (lobo_batch_log)
};

lobo_batch* lobo_batch_create(const rlm_config* cfg) {
  lobo_batch* b = new lobo_batch();
  b->c = *cfg;
  bool dbl = (cfg->algorithm == RLM_ALGO_DOUBLE_Q_LEARN);
  b->th_a.assign(cfg->memory_size, 0.0); b->d_a.assign(cfg->memory_size, 0.0);
  if (dbl) { b->th_b.assign(cfg->memory_size, 0.0); b->d_b.assign(cfg->memory_size, 0.0); }
  for (int i = 0; i < cfg->n_envs; ++i) {
    rlm_config one = *cfg;
    one.memory_size = cfg->memory_size;
    lobo_env* e = new lobo_env();
    e->sh_a = &b->th_a; e->sh_da = &b->d_a;
    if (dbl) { e->sh_b = &b->th_b; e->sh_db = &b->d_b; }
    e->init(&one, cfg->env_index0 + i);
    b->envs.push_back(e);
  }
  return b;
}
void lobo_batch_destroy(lobo_batch* b) { for (auto* e : b->envs) delete e; delete b; }

// phase A of one tick for every env: msgs[env]; step records (if recs) are written at recs[env*rec_cap + count[env]]
void lobo_batch_accumulate(lobo_batch* b, const rlm_tick_msg* msgs, rlm_step_record* recs, int32_t* rec_count, int32_t rec_cap) {
  b->pending.clear();
  b->log.clear();
  for (size_t i = 0; i < b->envs.size(); ++i) {
    rlm_step_record* r = nullptr;
    if (recs && rec_count[i] < rec_cap) r = &recs[i * (size_t)rec_cap + rec_count[i]];
    if (b->envs[i]->tick_deferred(msgs[i], r)) { b->pending.push_back((int)i); if (r) rec_count[i]++; }
  }
}
double* lobo_batch_dtheta(lobo_batch* b, int table) { return table == 0 ? b->d_a.data() : (b->d_b.empty() ? nullptr : b->d_b.data()); }
double* lobo_batch_theta(lobo_batch* b, int table) { return table == 0 ? b->th_a.data() : (b->th_b.empty() ? nullptr : b->th_b.data()); }
// phase B: theta += dtheta; dtheta = 0; pending envs select their next action under the new theta
void lobo_batch_apply(lobo_batch* b) {
  for (size_t i = 0; i < b->th_a.size(); ++i) { b->th_a[i] += b->d_a[i]; b->d_a[i] = 0.0; }
  for (size_t i = 0; i < b->th_b.size(); ++i) { b->th_b[i] += b->d_b[i]; b->d_b[i] = 0.0; }
  for (int i : b->pending) b->envs[i]->begin_step();
  b->pending.clear();
}
void lobo_batch_log(lobo_batch* b, int on) {
  b->log.clear();
  for (auto* e : b->envs) e->contrib_log = on ? &b->log : nullptr;
}
const lobo_contrib* lobo_batch_log_entries(lobo_batch* b, int64_t* n) {
  *n = (int64_t)b->log.size();
  return b->log.data();
}
int64_t lobo_batch_steps(lobo_batch* b) { int64_t s = 0; for (auto* e : b->envs) s += e->total_steps; return s; }
int64_t lobo_batch_sum_traces(lobo_batch* b) { int64_t s = 0; for (auto* e : b->envs) s += e->sum_traces; return s; }
void lobo_batch_stats(lobo_batch* b, int32_t env, rlm_env_stats* out) { lobo_stats(b->envs[env], out); }

int32_t lobo_to_ticks(const rlm_config* cfg, double px) { Venue v{}; v.init(cfg); return v.ToTicks(px); }
double lobo_to_price(const rlm_config* cfg, int32_t ticks) { Venue v{}; v.init(cfg); return v.ToPrice(ticks); }
double lobo_tick_size(const rlm_config* cfg, double px) { Venue v; v.init(cfg); return v.tick_size(px); }

void lobo_tiles(const rlm_config* cfg, const float* vars, int32_t* out) {
  State s;
  s.init(cfg->memory_size, cfg->n_actions, cfg->n_tilings);
  s.vars.assign(vars, vars + cfg->n_state_vars);
  s.populate();
  for (int a = 0; a < cfg->n_actions; ++a)
    for (int i = 0; i < 3 * cfg->n_tilings; ++i) out[a * 3 * cfg->n_tilings + i] = s.features[a][i];
}

void lobo_order_script(int64_t size, int64_t q_head, const rlm_order_op* ops, int32_t n_ops, rlm_order_state* out) {
  Order o;
  o.create(1.0, size, q_head);
  for (int i = 0; i < n_ops; ++i) {
    long ret = 0;
    switch (ops[i].op) {
      case 0: ret = o.doTransaction(ops[i].arg); break;
      case 1: o.doCancellation(ops[i].arg); break;
      case 2: o.addVolumeBehind(ops[i].arg); break;
      case 3: o.clearQueues(); break;
    }
    out[i].size = o.size; out[i].q_head = o.q_head; out[i].q_tail = o.q_tail;
    out[i].executed = o.total_executed; out[i].ret = ret;
  }
}

void lobo_rolling_mean(int32_t window, const double* vals, int32_t n, double* out) {
  RollingMean r;
  r.init(window);
  for (int i = 0; i < n; ++i) { r.push(vals[i]); out[2 * i] = r.mean(); out[2 * i + 1] = r.var(); }
}

uint64_t lobo_mt19937_64(uint64_t seed, int32_t n_skip) { MT64 g; g.seed(seed); uint64_t v = 0; for (int i = 0; i <= n_skip; ++i) v = g.next(); return v; }
int32_t lobo_glibc_rand(uint32_t seed, int32_t n_skip) { GlibcRand g; g.seed(seed); int32_t v = 0; for (int i = 0; i <= n_skip; ++i) v = g.next(); return v; }
double lobo_uniform_real(uint64_t seed, int32_t n_skip) { MT64 g; g.seed(seed); double v = 0; for (int i = 0; i <= n_skip; ++i) v = uniform_real01(g); return v; }
uint32_t lobo_uniform_int(uint64_t seed, uint32_t n, int32_t n_skip) { MT64 g; g.seed(seed); uint32_t v = 0; for (int i = 0; i <= n_skip; ++i) v = uniform_int_n(g, n); return v; }

void lobo_book_script(const lobo_book_op* ops, int32_t n_ops, lobo_book_result* out) {
  Side ask, bid;
  ask.is_ask = true; bid.is_ask = false;
  ask.Reset(); bid.Reset();
  Tx pending;  // op 6 sets the prints handed to the following ApplyChanges calls (book.cpp:67,94-95)
  for (int i = 0; i < n_ops; ++i) {
    const lobo_book_op& op = ops[i];
    Side& s = op.side == 0 ? ask : bid;
    lobo_book_result& r = out[i];
    memset(&r, 0, sizeof(r));
    r.r_ok = 1;
    try {
      switch (op.op) {
        case 0: {
          s.depth = op.n;
          long v[RLM_DEPTH];
          for (int l = 0; l < op.n; ++l) v[l] = op.vol[l];
          s.StashState();
          s.ApplyChanges(op.px, v, pending);
          break;
        }
        case 1: r.r_ok = s.PlaceOrder(op.a, op.b) ? 1 : 0; break;
        case 2: {
          Tx tx; tx.n = op.n;
          for (int k = 0; k < op.n; ++k) { tx.px[k] = op.px[k]; tx.vol[k] = op.vol[k]; }
          long v; s.ApplyTransactions(tx, op.a, v, r.r_proxy, r.r_value); r.r_volume = v;
          break;
        }
        case 3: { long v; adverse_selection(ask, bid, v, r.r_proxy, r.r_value); r.r_volume = v; break; }
        case 4: { long v; s.WalkTheBook(op.a, op.b, v, r.r_proxy, r.r_value); r.r_volume = v; break; }
        case 5: s.CancelAll(); break;
        case 6: pending.n = op.n; for (int k = 0; k < op.n; ++k) { pending.px[k] = op.px[k]; pending.vol[k] = op.vol[k]; } break;
      }
    } catch (const std::exception&) { r.r_ok = -1; }
    r.n_transacted = s.n_transacted_;
    if (s.o.live) { r.order.exists = 1; r.order.price = s.o.price; r.order.q_head = s.o.q_head; r.order.q_tail = s.o.q_tail; r.order.executed = s.o.total_executed; }
    r.obs_value = s.observed_value_; r.obs_volume = s.observed_volume_; r.total_volume = s.total_volume_;
  }
}

}  // extern "C"
