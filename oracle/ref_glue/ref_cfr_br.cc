// TEST INFRASTRUCTURE ONLY (NOT reference code): a C ABI over the unmodified reference's CFRBRSolver (algorithms/cfr_br.h)
// and TabularBestResponse (algorithms/best_response.h) for tests/cfr_br_lib.py, built by oracle/ref_cfr_br.mk into
// oracle/_ref/libspiel_ref_cfr_br.so.  It links against _ref/libspiel_ref_c.so, so games come from ref_load_game there and
// a process that loads both holds one copy of the reference.
#include <algorithm>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "open_spiel/algorithms/best_response.h"
#include "open_spiel/algorithms/cfr.h"
#include "open_spiel/algorithms/cfr_br.h"
#include "open_spiel/algorithms/expected_returns.h"
#include "open_spiel/algorithms/tabular_exploitability.h"
#include "open_spiel/policy.h"
#include "open_spiel/spiel.h"

using open_spiel::Game;
using open_spiel::algorithms::CFRBRSolver;

namespace {
struct GameHolder { std::shared_ptr<const Game> game; };   // the handle ref_load_game (ref_c_api.cc) returns
thread_local std::string g_err;

int CopyStr(const std::string& s, char* buf, int cap) {
  int n = (int)s.size();
  if (buf && cap > 0) { int m = n < cap - 1 ? n : cap - 1; memcpy(buf, s.data(), m); buf[m] = 0; }
  return n;
}
}  // namespace

// SpielFatalError throws (the handler ref_c_api.cc installs when libspiel_ref_c.so loads).
#define GUARD(stmt, onerr) try { stmt; } catch (const std::exception& e) { g_err = e.what(); onerr; }

extern "C" {

const char* ref_cfrbr_last_error() { return g_err.c_str(); }

void* ref_cfrbr_new(void* g) { GUARD(return new CFRBRSolver(*((GameHolder*)g)->game), return nullptr); }
void ref_cfrbr_free(void* c) { delete (CFRBRSolver*)c; }
int ref_cfrbr_iterate(void* c, int iters) {
  GUARD(for (int i = 0; i < iters; ++i) ((CFRBRSolver*)c)->EvaluateAndUpdatePolicy(); return 0, return 1);
}
// Table entry for an info-state key: copies up to cap values of each array; returns the number of legal actions, -1 if absent.
int ref_cfrbr_get(void* c, const char* key, int64_t* legal, double* regrets, double* cum_policy, double* cur_policy, int cap) {
  auto& table = ((CFRBRSolver*)c)->InfoStateValuesTable();
  auto it = table.find(key);
  if (it == table.end()) return -1;
  const auto& v = it->second;
  int n = (int)v.legal_actions.size();
  for (int i = 0; i < n && i < cap; ++i) {
    legal[i] = v.legal_actions[i];
    regrets[i] = v.cumulative_regrets[i];
    cum_policy[i] = v.cumulative_policy[i];
    cur_policy[i] = v.current_policy[i];
  }
  return n;
}
// All keys, '\n'-separated (sorted).
int ref_cfrbr_keys(void* c, char* buf, int cap) {
  auto& table = ((CFRBRSolver*)c)->InfoStateValuesTable();
  std::vector<std::string> keys;
  for (auto& kv : table) keys.push_back(kv.first);
  std::sort(keys.begin(), keys.end());
  std::string s;
  for (auto& k : keys) { s += k; s += '\n'; }
  return CopyStr(s, buf, cap);
}
int ref_cfrbr_serialize(void* c, char* buf, int cap) { GUARD(return CopyStr(((CFRBRSolver*)c)->Serialize(), buf, cap), return -1); }
void* ref_cfrbr_deserialize(const char* text) {
  GUARD(return open_spiel::algorithms::DeserializeCFRBRSolver(text).release(), return nullptr);
}
// NashConv, Exploitability and ExpectedReturns (depth_limit -1) of the average policy: out = {nash_conv, exploitability,
// expected return p0, expected return p1}.
int ref_cfrbr_average_eval(void* g, void* c, double* out) {
  const Game& game = *((GameHolder*)g)->game;
  auto* solver = (CFRBRSolver*)c;
  GUARD(auto avg = solver->AveragePolicy();
        out[0] = open_spiel::algorithms::NashConv(game, *avg);
        out[1] = open_spiel::algorithms::Exploitability(game, *avg);
        auto r = open_spiel::algorithms::ExpectedReturns(*game.NewInitialState(), *avg, -1);
        out[2] = r[0]; out[3] = r[1];
        return 0, return 1);
}
// TabularBestResponse(game, player, policy).GetBestResponseActions() and .Value(initial state) on a TabularPolicy given as
// n_keys information states ('\n'-separated keys; counts[i] (legal action, probability) pairs each, concatenated):
// actions[i] = the action chosen at key i, -1 where key i is not the player's.
int ref_tabular_br(void* g, int player, const char* keys, const int* counts, const int64_t* legal, const double* probs,
                   int n_keys, int64_t* actions, double* value) {
  const Game& game = *((GameHolder*)g)->game;
  std::unordered_map<std::string, open_spiel::ActionsAndProbs> table;
  std::vector<std::string> names;
  const char* k = keys;
  for (int i = 0, off = 0; i < n_keys; ++i) {
    const char* e = strchr(k, '\n');
    std::string key(k, e ? e - k : strlen(k));
    k = e ? e + 1 : k + key.size();
    open_spiel::ActionsAndProbs ap;
    for (int j = 0; j < counts[i]; ++j) ap.push_back({legal[off + j], probs[off + j]});
    off += counts[i];
    table[key] = ap;
    names.push_back(key);
  }
  GUARD(open_spiel::TabularPolicy policy(table);
        open_spiel::algorithms::TabularBestResponse br(game, player, &policy);
        auto best = br.GetBestResponseActions();
        for (int i = 0; i < n_keys; ++i) { auto it = best.find(names[i]); actions[i] = it == best.end() ? -1 : it->second; }
        *value = br.Value(*game.NewInitialState());
        return 0, return 1);
}

}  // extern "C"
