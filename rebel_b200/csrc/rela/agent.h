// A ReBeL agent played from outside (cfrb_agent_*, include/cfrb200.h): one handle's agent at `tables` independent tables, each a
// game against an external player, advanced one action per call.  The agent owns its handle, like play_lbr.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/cfrb200.h"
#include "cfrb_owner.h"
#include "params.h"

namespace rela {

class Agent {
 public:
  // policy: CFRB_MATCH_AVERAGE / _SAMPLED / _EVERY_NODE; w: flat Net2 weights (empty: none installed)
  Agent(const liars_dice::RecursiveSolvingParams& cfg, int device, int tables, int policy, uint64_t seed, const std::vector<float>& w)
      : tables_(tables), h_(open_handle(liars_dice::solver_config(cfg, device, tables))) {
    A_ = cfrb_num_actions(h_.get());
    H_ = cfrb_num_hands(h_.get());
    if (!w.empty()) check(cfrb_set_weights(h_.get(), w.data(), w.size(), 1), "cfrb_set_weights");
    cfrb_agent* a = nullptr;
    check(cfrb_agent_create(h_.get(), tables, seed, policy, &a), "cfrb_agent_create");
    a_.reset(a);
  }

  // A blueprint agent: the compact full-tree table `strategy` [N - 1][H] (its size checked by the caller) uploaded to `device`
  // with cfrb_blueprint_create's checks plays at every table; it never solves and needs no handle.
  Agent(int num_dice, int num_faces, const std::vector<double>& strategy, int device, int tables, uint64_t seed) : tables_(tables) {
    A_ = 1 + 2 * num_dice * num_faces;
    H_ = 1;
    for (int i = 0; i < num_dice; ++i) H_ *= num_faces;
    cfrb_blueprint* b = nullptr;
    check(cfrb_blueprint_create(device, num_dice, num_faces, strategy.data(), &b), "cfrb_blueprint_create");
    bp_.reset(b);
    cfrb_agent* a = nullptr;
    check(cfrb_agent_create_blueprint(bp_.get(), tables, seed, &a), "cfrb_agent_create_blueprint");
    a_.reset(a);
  }

  void close() {   // the agent first: it reads its handle (or blueprint) when it is destroyed
    a_.reset();
    bp_.reset();
    h_.reset();
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
  int tables_ = 0, A_ = 0, H_ = 0;
  HandlePtr h_;
  BlueprintPtr bp_;
  AgentPtr a_;   // declared after its handle and blueprint: released first

  cfrb_agent* live() {
    if (!a_) throw std::runtime_error("Agent: closed");
    return a_.get();
  }
  int size(const std::vector<int32_t>& ids, const char* who) const {
    if ((int64_t)ids.size() > tables_)
      throw std::runtime_error(std::string(who) + ": more ids than tables (" + std::to_string(tables_) + ")");
    return (int)ids.size();
  }
};

}  // namespace rela
