// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// extern "C" wrappers around the reference's evaluation functions that recursive_eval reports (recursive_eval.cc:270-425):
// compute_ev2, compute_immediate_regrets and the fictitious-play sampled recursive strategy.  Compiled against the headers of a
// checkout of the original project and linked with oracle/_ref/libref_nofma.so, which holds the reference's own objects built
// with -ffp-contract=off (recipe: oracle/ev_regret.py build_ref(), output: oracle/_ref/libref_eval_nofma.so).  Used by
// oracle/make_golden_r3.py to generate tests/golden/ev_regrets.npz.  Nothing in rebel_b200/ links or dlopens it.
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "real_net.h"
#include "recursive_solving.h"
#include "subgame_solving.h"

using namespace liars_dice;

namespace {

thread_local std::string g_err;

TreeStrategy dense_to_tree_strategy(const Game& game, size_t N, const double* dense) {
  TreeStrategy s(N, std::vector<std::vector<double>>(game.num_hands(), std::vector<double>(game.num_actions(), 0.0)));
  size_t k = 0;
  for (auto& n : s)
    for (auto& h : n)
      for (double& v : h) v = dense[k++];
  return s;
}

}  // namespace

extern "C" {

const char* refev_last_error() { return g_err.c_str(); }

// compute_ev2 (subgame_solving.cc:975-982) of two dense [N][H][A] full-tree strategies.
int refev_ev2(int D, int F, const double* s1, const double* s2, double* out2) {
  try {
    Game game(D, F);
    const size_t N = unroll_tree(game).size();
    auto e = compute_ev2(game, dense_to_tree_strategy(game, N, s1), dense_to_tree_strategy(game, N, s2));
    out2[0] = e[0];
    out2[1] = e[1];
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// compute_immediate_regrets (subgame_solving.cc:984-1050) of n dense [N][H][A] strategies: immediate_out [N][H].
int refev_immediate_regrets(int D, int F, const double* strategies, int n, double* immediate_out) {
  try {
    Game game(D, F);
    const size_t N = unroll_tree(game).size(), per = N * game.num_hands() * game.num_actions();
    std::vector<TreeStrategy> list;
    for (int i = 0; i < n; ++i) list.push_back(dense_to_tree_strategy(game, N, strategies + per * i));
    auto r = compute_immediate_regrets(game, list);
    size_t k = 0;
    for (auto& node : r)
      for (double v : node) immediate_out[k++] = v;
    return (int)N;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// compute_sampled_strategy_recursive_to_leaf (recursive_solving.cc:301-327) with fictitious play as the subgame solver
// (SubgameSolvingParams::use_cfr = false: recursive_eval without --cfr), zero value net.  strategy_out: dense [N_full][H][A].
int refev_sampled_strategy_fp(int D, int F, int num_iters, int max_depth, int linear_update, int seed, double* strategy_out) {
  try {
    Game game(D, F);
    const int H = game.num_hands(), A = game.num_actions();
    SubgameSolvingParams params;
    params.num_iters = num_iters;
    params.max_depth = max_depth;
    params.linear_update = linear_update != 0;
    params.use_cfr = false;
    auto strategy = compute_sampled_strategy_recursive_to_leaf(game, params, create_zero_net(H, false), seed);
    size_t k = 0;
    for (auto& n : strategy) {
      if (n.empty()) { k += (size_t)H * A; continue; }   // terminal nodes keep an empty entry
      for (auto& h : n)
        for (double v : h) strategy_out[k++] = v;
    }
    return (int)strategy.size();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

}  // extern "C"
