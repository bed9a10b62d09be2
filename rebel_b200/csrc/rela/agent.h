// A ReBeL agent played from outside (cfrb_agent_*, include/cfrb200.h): one handle's agent at `tables` independent tables, each a
// game against an external player, advanced one action per call.  The agent owns its handle, like play_lbr.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/cfrb200.h"
#include "params.h"

namespace rela {

class Agent {
 public:
  // policy: CFRB_MATCH_AVERAGE / CFRB_MATCH_SAMPLED; w: flat Net2 weights (empty: none installed)
  Agent(const liars_dice::RecursiveSolvingParams& cfg, int device, int tables, int policy, uint64_t seed, const std::vector<float>& w)
      : tables_(tables) {
    try {
      const cfrb_config c = liars_dice::solver_config(cfg, device, tables);
      check(cfrb_create(&c, &h_), "cfrb_create");
      A_ = cfrb_num_actions(h_);
      H_ = cfrb_num_hands(h_);
      if (!w.empty()) check(cfrb_set_weights(h_, w.data(), w.size(), 1), "cfrb_set_weights");
      check(cfrb_agent_create(h_, tables, seed, policy, &a_), "cfrb_agent_create");
    } catch (...) {
      close();
      throw;
    }
  }
  ~Agent() { close(); }
  Agent(const Agent&) = delete;
  Agent& operator=(const Agent&) = delete;

  void close() {
    if (a_) cfrb_agent_destroy(a_);
    if (h_) cfrb_destroy(h_);
    a_ = nullptr;
    h_ = nullptr;
  }

  int numActions() const { return A_; }
  int numHands() const { return H_; }
  int tables() const { return tables_; }

  void newGames(const std::vector<int32_t>& ids, const std::vector<int32_t>& seats, const std::vector<int32_t>& hands,
                const std::vector<uint64_t>& keys) {
    const int n = size(ids, "new_games");
    if ((int)seats.size() != n || (int)hands.size() != n || (!keys.empty() && (int)keys.size() != n))
      throw std::runtime_error("new_games: ids, seats, hands (and keys) must have the same length");
    check(cfrb_agent_new_games(live(), n, ids.data(), seats.data(), hands.data(), keys.empty() ? nullptr : keys.data()),
          "cfrb_agent_new_games");
  }

  // actions: in the action to apply or -1 (the agent plays), out the action played; probs [n][A]; done [n]
  void step(const std::vector<int32_t>& ids, std::vector<int32_t>& actions, std::vector<double>& probs, std::vector<int32_t>& done) {
    const int n = size(ids, "step");
    if ((int)actions.size() != n) throw std::runtime_error("step: ids and actions must have the same length");
    probs.resize((size_t)n * A_);
    done.resize(n);
    check(cfrb_agent_step(live(), n, ids.data(), actions.data(), probs.data(), done.data()), "cfrb_agent_step");
  }

  std::vector<double> policy(const std::vector<int32_t>& ids) {
    const int n = size(ids, "policy");
    std::vector<double> out((size_t)n * H_ * A_);
    check(cfrb_agent_policy(live(), n, ids.data(), out.data()), "cfrb_agent_policy");
    return out;
  }

  struct State {
    std::vector<int32_t> last_bid, player, ply, subgames, act_iteration;
    std::vector<double> root_beliefs;
  };
  State state(const std::vector<int32_t>& ids) {
    const int n = size(ids, "state");
    State s;
    for (auto* v : {&s.last_bid, &s.player, &s.ply, &s.subgames, &s.act_iteration}) v->resize(n);
    s.root_beliefs.resize((size_t)n * 2 * H_);
    check(cfrb_agent_state(live(), n, ids.data(), s.last_bid.data(), s.player.data(), s.ply.data(), s.subgames.data(),
                           s.act_iteration.data(), s.root_beliefs.data()),
          "cfrb_agent_state");
    return s;
  }

  // subgames solved, iterations run for them, device ms of the solves
  void counts(int64_t* solves, int64_t* subgame_iters, double* solve_ms) {
    check(cfrb_agent_counts(live(), solves, subgame_iters), "cfrb_agent_counts");
    check(cfrb_agent_solve_ms(live(), solve_ms), "cfrb_agent_solve_ms");
  }

 private:
  cfrb_handle* h_ = nullptr;
  cfrb_agent* a_ = nullptr;
  int tables_ = 0, A_ = 0, H_ = 0;

  static void check(int rc, const char* what) {
    if (rc < 0) throw std::runtime_error(std::string(what) + ": " + cfrb_last_error());
  }
  cfrb_agent* live() {
    if (!a_) throw std::runtime_error("Agent: closed");
    return a_;
  }
  int size(const std::vector<int32_t>& ids, const char* who) const {
    if ((int64_t)ids.size() > tables_)
      throw std::runtime_error(std::string(who) + ": more ids than tables (" + std::to_string(tables_) + ")");
    return (int)ids.size();
  }
};

}  // namespace rela
