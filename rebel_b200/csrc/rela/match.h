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
  double seconds = 0;
};

// One handle per agent; `games` games, `slots` of them at a time.  policy: CFRB_MATCH_AVERAGE / CFRB_MATCH_SAMPLED.
inline MatchResult play_match(const liars_dice::RecursiveSolvingParams& cfg_a, const liars_dice::RecursiveSolvingParams& cfg_b,
                              int device, int games, uint64_t seed, int policy, const std::vector<float>& w_a,
                              const std::vector<float>& w_b, int slots) {
  if (games < 2) throw std::runtime_error("play_match: games must be >= 2");
  slots = std::max(1, std::min(slots, games));
  cfrb_handle* h[2] = {nullptr, nullptr};
  cfrb_match* m = nullptr;
  auto cleanup = [&]() {
    if (m) cfrb_match_destroy(m);
    for (auto* x : h) if (x) cfrb_destroy(x);
  };
  auto check = [&](int rc, const char* what) {
    if (rc < 0) {
      const std::string err = std::string(what) + ": " + cfrb_last_error();
      cleanup();
      throw std::runtime_error(err);
    }
    return rc;
  };
  const liars_dice::RecursiveSolvingParams* cfgs[2] = {&cfg_a, &cfg_b};
  const std::vector<float>* ws[2] = {&w_a, &w_b};
  for (int k = 0; k < 2; ++k) {
    const cfrb_config c = liars_dice::solver_config(*cfgs[k], device, slots);
    check(cfrb_create(&c, &h[k]), "cfrb_create");
    if (!ws[k]->empty()) check(cfrb_set_weights(h[k], ws[k]->data(), ws[k]->size(), 1), "cfrb_set_weights");
  }
  check(cfrb_match_create(h[0], h[1], slots, games, seed, policy, &m), "cfrb_match_create");
  MatchResult r;
  const auto t0 = std::chrono::steady_clock::now();
  while (check(cfrb_match_run(m, 8, nullptr), "cfrb_match_run") > 0) {
  }
  r.payoff.resize(games);
  r.plies.resize(games);
  check(cfrb_match_results(m, r.payoff.data(), r.plies.data(), &r.solves, &r.subgame_iters), "cfrb_match_results");
  r.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  cleanup();
  return r;
}

struct LbrResult : MatchResult {
  int64_t whatif_solves = 0, deferred_slot_rounds = 0;
  int capacity = 0;
};

// Default subgames per round of a local-best-response run: two per slot (a slot asks for one subgame at a game start or a
// pseudo-leaf and for one per legal raise at an LBR decision on the edge of the agent's subgame), at least A - 1.
inline int lbr_default_capacity(int slots, int num_actions) { return std::max(2 * slots, num_actions - 1); }

// Local best response against one agent (cfrb_match_create_lbr): `games` games, `slots` at a time; payoff[] is the agent's.
// max_subgames = 0 takes lbr_default_capacity.
inline LbrResult play_lbr(const liars_dice::RecursiveSolvingParams& cfg, int device, int games, uint64_t seed, const std::vector<float>& w,
                          int slots, int max_subgames) {
  if (games < 2) throw std::runtime_error("play_lbr: games must be >= 2");
  slots = std::max(1, std::min(slots, games));
  cfrb_handle* h = nullptr;
  cfrb_match* m = nullptr;
  auto cleanup = [&]() {
    if (m) cfrb_match_destroy(m);
    if (h) cfrb_destroy(h);
  };
  auto check = [&](int rc, const char* what) {
    if (rc < 0) {
      const std::string err = std::string(what) + ": " + cfrb_last_error();
      cleanup();
      throw std::runtime_error(err);
    }
    return rc;
  };
  LbrResult r;
  if (max_subgames <= 0) {                           // the game's number of actions, from a one-subgame handle
    const cfrb_config c1 = liars_dice::solver_config(cfg, device, 1);
    check(cfrb_create(&c1, &h), "cfrb_create");
    max_subgames = lbr_default_capacity(slots, cfrb_num_actions(h));
    cfrb_destroy(h);
    h = nullptr;
  }
  r.capacity = max_subgames;
  const cfrb_config c = liars_dice::solver_config(cfg, device, max_subgames);
  check(cfrb_create(&c, &h), "cfrb_create");
  if (!w.empty()) check(cfrb_set_weights(h, w.data(), w.size(), 1), "cfrb_set_weights");
  check(cfrb_match_create_lbr(h, slots, games, seed, &m), "cfrb_match_create_lbr");
  const auto t0 = std::chrono::steady_clock::now();
  while (check(cfrb_match_run(m, 8, nullptr), "cfrb_match_run") > 0) {
  }
  r.payoff.resize(games);
  r.plies.resize(games);
  check(cfrb_match_results(m, r.payoff.data(), r.plies.data(), &r.solves, &r.subgame_iters), "cfrb_match_results");
  check(cfrb_match_lbr_counts(m, &r.whatif_solves, &r.deferred_slot_rounds), "cfrb_match_lbr_counts");
  r.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  cleanup();
  return r;
}

}  // namespace rela
