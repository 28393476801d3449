// rlm_ingest.cpp -- reference-format CSV pair -> packed rlm_tick_msg stream (host code, no GPU needed).
//
// Restates what the reference's data layer hands to Intraday::NextState, one message sequence per tick:
//   * market depth rows      data::basic::MarketDepth        src/data/basic.cpp:20-108   (22 columns; a row with a
//                            non-positive price is skipped; date, HH:MM:SS.mmm, AP1..5, AV1..5, BP1..5, BV1..5)
//   * time and sales         data::basic::TimeAndSales       src/data/basic.cpp:112-202  (date, time, price, size; prints
//                            with non-positive price or size are dropped)
//   * which prints belong to a tick   Streamer::LoadUntil    src/data/streamer.cpp:57-81: everything not consumed yet
//                            whose time is <= the time of the tick's (first) depth row, aggregated by the 4-decimal
//                            price key of utilities/comparison.h:13-16 (the first price seen for a key is the map's key)
//   * which depth rows belong to a tick   Intraday::UpdateBookProfiles  src/environment/intraday.cpp:274-313: rows are
//                            applied while the NEXT row carries the same timestamp (WillTimeChange) or the book state is
//                            invalid (BookUtils::IsValidState, src/market/book.cpp:612-625)
// Numbers are parsed with strtof / strtol exactly like the reference's stof / stol / stoi.
// A tick is emitted as [RLM_TICK_TX_MORE messages] + [rows flagged RLM_TICK_PARTIAL] + one last row (include/rlm_flow.h).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "rlm.h"

namespace {

struct MdRow { int date; long time; float ap[5], bp[5]; long av[5], bv[5]; };
struct Print { int date; long time; float px; long size; };

void split(const std::string& line, std::vector<std::string>& cols) {  // CSV::parseRow, src/utilities/csv.cpp:30-45
  cols.clear();
  size_t pos = 0;
  while (true) {
    size_t next = line.find(',', pos);
    if (next == std::string::npos) { cols.push_back(line.substr(pos)); break; }
    cols.push_back(line.substr(pos, next - pos));
    pos = next + 1;
  }
}
long to_time(const std::string& s) {  // string_to_time, include/utilities/time.h:28-39: fixed offsets HH:MM:SS.mmm
  if (s.size() < 12) return -1;
  auto num = [&](size_t a, size_t n) { return strtol(s.substr(a, n).c_str(), nullptr, 10); };
  return ((num(0, 2) * 60 + num(3, 2)) * 60 + num(6, 2)) * 1000 + num(9, 3);
}
bool read_lines(const char* path, std::vector<std::string>& out, std::string& err) {
  FILE* f = fopen(path, "rb");
  if (!f) { err = std::string("cannot open ") + path; return false; }
  std::string cur;
  char buf[1 << 16];
  size_t n;
  bool first = true;
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) {
    for (size_t i = 0; i < n; ++i) {
      if (buf[i] == '\n') {
        if (!first) out.push_back(cur);  // csv_.skip(1): the header line is ignored (basic.cpp:25,131)
        first = false;
        cur.clear();
      } else cur.push_back(buf[i]);
    }
  }
  if (!cur.empty() && !first) out.push_back(cur);
  fclose(f);
  return true;
}
double pkey(double p) { return rint(p * 10000.0); }

}  // namespace

extern "C" const char* rlm_last_error(void);
int fail(int code, const std::string& msg);  // rlm_handle.h

extern "C" int rlm_ingest_csv(const char* md_path, const char* tas_path, rlm_tick_msg* out, int64_t cap, int64_t* n_msgs, int64_t* n_ticks) {
  if (!md_path || !tas_path || !n_msgs) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_ingest_csv: null argument");
  std::string err;
  std::vector<std::string> lines, cols;
  std::vector<MdRow> rows;
  if (!read_lines(md_path, lines, err)) return fail(RLM_ERR_INVALID_ARGUMENT, err);
  std::vector<std::string> piece;
  cols.clear();
  for (const std::string& ln : lines) {
    // MarketDepth::_LoadRow (basic.cpp:30-43) keeps APPENDING the columns of further lines to its row buffer until it
    // holds exactly 22: after a line of any other width the buffer never matches again and the data ends there.
    // Reproduced, not repaired.
    split(ln, piece);
    cols.insert(cols.end(), piece.begin(), piece.end());
    if (cols.size() != 22) continue;
    MdRow r;
    r.date = (int)strtol(cols[0].c_str(), nullptr, 10);
    r.time = to_time(cols[1]);
    bool ok = true;
    for (int i = 0; i < 5 && ok; ++i) {
      r.ap[i] = strtof(cols[2 + i].c_str(), nullptr);
      r.bp[i] = strtof(cols[12 + i].c_str(), nullptr);
      if ((double)r.ap[i] <= 0.0 || (double)r.bp[i] <= 0.0) { ok = false; break; }  // basic.cpp:54-58: the row is dropped
      r.av[i] = strtol(cols[7 + i].c_str(), nullptr, 10);
      r.bv[i] = strtol(cols[17 + i].c_str(), nullptr, 10);
    }
    if (ok) rows.push_back(r);
    cols.clear();
  }
  lines.clear();
  std::vector<Print> prints;
  if (!read_lines(tas_path, lines, err)) return fail(RLM_ERR_INVALID_ARGUMENT, err);
  cols.clear();
  for (const std::string& ln : lines) {
    split(ln, piece);  // TimeAndSales::_LoadRow (basic.cpp:136-148): same buffer behaviour, 4 columns
    cols.insert(cols.end(), piece.begin(), piece.end());
    if (cols.size() != 4) continue;
    Print p;
    p.date = (int)strtol(cols[0].c_str(), nullptr, 10);
    p.time = to_time(cols[1]);
    p.px = strtof(cols[2].c_str(), nullptr);
    p.size = strtol(cols[3].c_str(), nullptr, 10);
    if ((double)p.px > 0.0 && p.size > 0) prints.push_back(p);  // basic.cpp:158-159
    cols.clear();
  }
  // the packed levels are "best first": the reference's books sort by price, the stream contract requires it
  for (size_t i = 0; i < rows.size(); ++i)
    for (int l = 1; l < 5; ++l)
      if (!(pkey(rows[i].ap[l]) > pkey(rows[i].ap[l - 1])) || !(pkey(rows[i].bp[l]) < pkey(rows[i].bp[l - 1])))
        return fail(RLM_ERR_UNSUPPORTED, "rlm_ingest_csv: depth row " + std::to_string(i) + " is not strictly ordered best-first (AP ascending, BP descending)");

  int64_t n_out = 0, ticks = 0;
  auto emit = [&](const rlm_tick_msg& m) { if (out && n_out < cap) out[n_out] = m; ++n_out; };
  size_t j = 0;  // next unconsumed print
  bool have_stash = false;
  double stash_mid = 0.0;  // midprice of the book the tick started from (last_price(0) of both sides)
  size_t i = 0;
  while (i < rows.size()) {
    const MdRow& first = rows[i];
    // ---- prints of the tick: time <= the first row's time (NextState's target, intraday.cpp:227-231)
    std::vector<std::pair<float, long>> agg;  // (first price seen for the key, volume), kept in key order
    while (j < prints.size() && (prints[j].date < first.date || (prints[j].date == first.date && prints[j].time <= first.time))) {
      const double k = pkey(prints[j].px);
      size_t a = 0;
      while (a < agg.size() && pkey(agg[a].first) < k) ++a;
      if (a < agg.size() && pkey(agg[a].first) == k) agg[a].second += prints[j].size;
      else agg.insert(agg.begin() + a, std::make_pair(prints[j].px, prints[j].size));
      ++j;
    }
    if (agg.size() > RLM_TX_CAP)
      return fail(RLM_ERR_UNSUPPORTED, "rlm_ingest_csv: more than " + std::to_string(RLM_TX_CAP) + " distinct print prices in the tick of depth row " + std::to_string(i));
    // all but the last RLM_N_TX_MAX prices travel ahead in RLM_TICK_TX_MORE messages
    size_t lead = agg.size() > RLM_N_TX_MAX ? agg.size() - RLM_N_TX_MAX : 0, a = 0;
    while (a < lead) {
      rlm_tick_msg m;
      memset(&m, 0, sizeof(m));
      m.flags = RLM_TICK_TX_MORE;
      m.date = first.date; m.time_ms = (int32_t)first.time;
      int n = 0;
      while (a < lead && n < RLM_N_TX_MAX) { m.tx_px[n] = agg[a].first; m.tx_vol[n] = (int32_t)agg[a].second; ++n; ++a; }
      m.n_tx = n;
      emit(m);
    }
    // ---- depth rows of the tick
    while (true) {
      const MdRow& r = rows[i];
      rlm_tick_msg m;
      memset(&m, 0, sizeof(m));
      for (int l = 0; l < 5; ++l) {
        m.ask_px[l] = r.ap[l]; m.bid_px[l] = r.bp[l];
        m.ask_vol[l] = (int32_t)r.av[l]; m.bid_vol[l] = (int32_t)r.bv[l];
      }
      int n = 0;
      for (size_t b = lead; b < agg.size(); ++b) { m.tx_px[n] = agg[b].first; m.tx_vol[n] = (int32_t)agg[b].second; ++n; }
      m.n_tx = n;
      m.date = r.date; m.time_ms = (int32_t)r.time;
      bool more = false;
      if (i + 1 < rows.size()) {
        if (rows[i + 1].time == r.time) more = true;  // !WillTimeChange (streamer.cpp:116-119; compares times only)
        else if (have_stash) {                          // BookUtils::IsValidState (book.cpp:612-625)
          const double mp = ((double)r.ap[0] + (double)r.bp[0]) / 2.0;
          const bool valid = ((double)r.ap[0] - (double)r.bp[0] >= 0.0) && (mp > 0.0) && (fabs(mp - stash_mid) < mp);
          if (!valid) more = true;
        }
      }
      m.flags = more ? RLM_TICK_PARTIAL : 0;
      emit(m);
      ++i;
      if (!more) break;
    }
    // the next tick stashes the book this one ended with
    have_stash = true;
    stash_mid = ((double)rows[i - 1].ap[0] + (double)rows[i - 1].bp[0]) / 2.0;
    ++ticks;
  }
  *n_msgs = n_out;
  if (n_ticks) *n_ticks = ticks;
  if (out && n_out > cap) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_ingest_csv: output buffer too small");
  return RLM_OK;
}
