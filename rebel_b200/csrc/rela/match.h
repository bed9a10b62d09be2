// Head-to-head evaluation of two ReBeL agents (cfrb_match_*, include/cfrb200.h): each agent is a RecursiveSolvingParams plus a
// value net; both re-solve subgames only along the path actually played, so the cost per game does not depend on the size of
// the game tree and games the full-tree evaluators refuse (2x5f, 2x6f, 1x17f, ...) can be evaluated.
#pragma once
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/cfrb200.h"
#include "cfrb_owner.h"
#include "params.h"

namespace rela {

// Mean payoff to agent A and its standard error over the seat-swapped pairs (games 2i, 2i+1 share the deal: their mean is one
// sample), and A's mean payoff in seat 0 (even games) and seat 1 (odd games).
struct MatchStats { double mean = 0, stderr_ = 0, seat[2] = {0, 0}; };
inline MatchStats match_stats(const std::vector<float>& payoff) {
  const size_t n = payoff.size() / 2;
  if (n == 0) throw std::runtime_error("match_stats: at least one pair of games is needed");
  MatchStats s;
  double sum = 0, s0 = 0, s1 = 0;
  for (size_t i = 0; i < n; ++i) {
    sum += 0.5 * ((double)payoff[2 * i] + (double)payoff[2 * i + 1]);
    s0 += payoff[2 * i]; s1 += payoff[2 * i + 1];
  }
  s.mean = sum / n;
  s.seat[0] = s0 / n; s.seat[1] = s1 / n;
  double ss = 0;
  for (size_t i = 0; i < n; ++i) {
    const double d = 0.5 * ((double)payoff[2 * i] + (double)payoff[2 * i + 1]) - s.mean;
    ss += d * d;
  }
  s.stderr_ = n > 1 ? std::sqrt(ss / (n - 1) / n) : std::numeric_limits<double>::infinity();
  return s;
}

struct MatchResult {
  std::vector<float> payoff;   // [games] to agent A
  std::vector<int> plies;      // [games]
  int64_t solves = 0, subgame_iters = 0;
  int64_t agent_solves[2] = {0, 0};   // subgames A and B solved
  double seconds = 0;
};

// A blueprint of cfg's game on `device` from a compact full-tree table [N - 1][H] (cfrb_blueprint_create's checks).
inline BlueprintPtr upload_blueprint(const liars_dice::RecursiveSolvingParams& cfg, int device, const std::vector<double>& table) {
  cfrb_blueprint* b = nullptr;
  check(cfrb_blueprint_create(device, cfg.num_dice, cfg.num_faces, table.data(), &b), "cfrb_blueprint_create");
  return BlueprintPtr(b);
}

// One handle per agent; `games` games, `slots` of them at a time.  policy (A's), policy_b: CFRB_MATCH_AVERAGE / _SAMPLED /
// _EVERY_NODE; a pair of different policies goes through cfrb_match_create2.  bp_a / bp_b (non-null): that agent is a blueprint
// of this compact table instead (no handle, its cfg and weights unused; cfrb_match_create3).
inline MatchResult play_match(const liars_dice::RecursiveSolvingParams& cfg_a, const liars_dice::RecursiveSolvingParams& cfg_b,
                              int device, int games, uint64_t seed, int policy, const std::vector<float>& w_a,
                              const std::vector<float>& w_b, int slots, int policy_b, const std::vector<double>* bp_a = nullptr,
                              const std::vector<double>* bp_b = nullptr) {
  if (games < 2) throw std::runtime_error("play_match: games must be >= 2");
  slots = std::max(1, std::min(slots, games));
  const liars_dice::RecursiveSolvingParams* cfgs[2] = {&cfg_a, &cfg_b};
  const std::vector<float>* ws[2] = {&w_a, &w_b};
  const std::vector<double>* bps[2] = {bp_a, bp_b};
  HandlePtr h[2];
  BlueprintPtr bp[2];
  for (int k = 0; k < 2; ++k) {
    if (bps[k]) {
      bp[k] = upload_blueprint(*cfgs[k], device, *bps[k]);
      continue;
    }
    h[k] = open_handle(liars_dice::solver_config(*cfgs[k], device, slots));
    if (!ws[k]->empty()) check(cfrb_set_weights(h[k].get(), ws[k]->data(), ws[k]->size(), 1), "cfrb_set_weights");
  }
  cfrb_match* raw = nullptr;
  if (bp[0] || bp[1]) {
    const cfrb_match_agent a{h[0].get(), bp[0].get(), policy}, b{h[1].get(), bp[1].get(), policy_b};
    check(cfrb_match_create3(&a, &b, slots, games, seed, &raw), "cfrb_match_create3");
  } else if (policy == policy_b) {
    check(cfrb_match_create(h[0].get(), h[1].get(), slots, games, seed, policy, &raw), "cfrb_match_create");
  } else {
    check(cfrb_match_create2(h[0].get(), h[1].get(), slots, games, seed, policy, policy_b, &raw), "cfrb_match_create2");
  }
  const MatchPtr m(raw);   // released before the handles and blueprints it reads
  MatchResult r;
  const auto t0 = std::chrono::steady_clock::now();
  while (check(cfrb_match_run(m.get(), 8, nullptr), "cfrb_match_run") > 0) {
  }
  r.payoff.resize(games);
  r.plies.resize(games);
  check(cfrb_match_results(m.get(), r.payoff.data(), r.plies.data(), &r.solves, &r.subgame_iters), "cfrb_match_results");
  check(cfrb_match_agent_solves(m.get(), r.agent_solves), "cfrb_match_agent_solves");
  r.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return r;
}

struct LbrResult : MatchResult {
  int64_t whatif_solves = 0, deferred_slot_rounds = 0;
  int capacity = 0;
};

// Default subgames per round of a local-best-response run: two per slot (a slot asks for one subgame at a game start or a
// pseudo-leaf and for one per legal raise at an LBR decision on the edge of the agent's subgame), at least A - 1.
inline int lbr_default_capacity(int slots, int num_actions) { return std::max(2 * slots, num_actions - 1); }

// Local best response against one agent playing `policy` (CFRB_MATCH_AVERAGE or CFRB_MATCH_EVERY_NODE; cfrb_match_create_lbr2):
// `games` games, `slots` at a time; payoff[] is the agent's.  max_subgames = 0 takes lbr_default_capacity.  bp (non-null): LBR
// against a blueprint of this compact table instead (cfrb_match_create_lbr_blueprint: no handle, no solves; capacity 0).
inline LbrResult play_lbr(const liars_dice::RecursiveSolvingParams& cfg, int device, int games, uint64_t seed, const std::vector<float>& w,
                          int slots, int max_subgames, int policy = CFRB_MATCH_AVERAGE, const std::vector<double>* bp = nullptr) {
  if (games < 2) throw std::runtime_error("play_lbr: games must be >= 2");
  slots = std::max(1, std::min(slots, games));
  LbrResult r;
  HandlePtr h;
  BlueprintPtr b;
  cfrb_match* raw = nullptr;
  if (bp) {
    b = upload_blueprint(cfg, device, *bp);
    check(cfrb_match_create_lbr_blueprint(b.get(), slots, games, seed, &raw), "cfrb_match_create_lbr_blueprint");
  } else {
    if (max_subgames <= 0) max_subgames = lbr_default_capacity(slots, 2 * cfg.num_dice * cfg.num_faces + 1);
    r.capacity = max_subgames;
    h = open_handle(liars_dice::solver_config(cfg, device, max_subgames));
    if (!w.empty()) check(cfrb_set_weights(h.get(), w.data(), w.size(), 1), "cfrb_set_weights");
    check(cfrb_match_create_lbr2(h.get(), slots, games, seed, policy, &raw), "cfrb_match_create_lbr2");
  }
  const MatchPtr m(raw);   // released before the handle or blueprint it reads
  const auto t0 = std::chrono::steady_clock::now();
  while (check(cfrb_match_run(m.get(), 8, nullptr), "cfrb_match_run") > 0) {
  }
  r.payoff.resize(games);
  r.plies.resize(games);
  check(cfrb_match_results(m.get(), r.payoff.data(), r.plies.data(), &r.solves, &r.subgame_iters), "cfrb_match_results");
  check(cfrb_match_lbr_counts(m.get(), &r.whatif_solves, &r.deferred_slot_rounds), "cfrb_match_lbr_counts");
  r.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return r;
}

}  // namespace rela
