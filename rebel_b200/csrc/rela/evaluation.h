// Evaluation entry points of the `rela` module — the reference's compute_exploitability_fp / compute_exploitability_with_net /
// compute_stats_with_net (rela/pybind.cc:45-104) and eval_net (stats.cc:44-153) — with every subgame solve batched on the GPU
// through the C ABI.  The value net of a checkpoint is used in two ways: as flat weights for the solver kernels
// (cfrb_set_weights) and, for the handful of single-row evaluations eval_net makes, through libtorch on the host.
#pragma once
#include <torch/script.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <functional>
#include <memory>
#include <numeric>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "../../../include/cfrb200.h"
#include "cfrb_owner.h"
#include "params.h"
#include "recursive_eval.h"

namespace rela {

// Net2 parameters of a TorchScript checkpoint, flattened in the order cfrb_set_weights expects (cfvpy/models.py:64-94).
inline std::vector<float> flat_weights_of(torch::jit::Module& m) {
  static const char* kOrder[] = {"body.0.weight", "body.0.bias", "body.1.weight", "body.1.bias", "body.4.weight",
                                 "body.4.bias",   "body.5.weight", "body.5.bias", "output.weight", "output.bias"};
  std::vector<float> flat;
  // only Net2(n_hidden=256, n_layers=2, use_layer_norm=True) is accelerated: any further parameter (a deeper body) is an error,
  // not something to drop silently
  for (const auto& p : m.named_parameters()) {
    bool known = false;
    for (const char* name : kOrder) known |= p.name == name;
    if (!known)
      throw std::runtime_error("value net has an unexpected parameter '" + p.name +
                               "': rebel_b200 accelerates Net2(n_hidden=256, n_layers=2, use_layer_norm=True) only");
    if (p.name == "body.0.weight" && (p.value.dim() != 2 || p.value.size(0) != 256))
      throw std::runtime_error("value net: n_hidden must be 256");
  }
  for (const char* name : kOrder) {
    bool found = false;
    for (const auto& p : m.named_parameters()) {
      if (p.name == name) {
        auto t = p.value.detach().to(torch::kCPU, torch::kFloat32).contiguous();
        flat.insert(flat.end(), t.data_ptr<float>(), t.data_ptr<float>() + t.numel());
        found = true;
        break;
      }
    }
    if (!found) throw std::runtime_error(std::string("value net is not a 2-layer LayerNorm Net2: missing parameter ") + name);
  }
  return flat;
}

// One subgame solver over the FULL tree from the initial state (build_solver(game, params), subgame_solving.h:119-134).
class FullTreeSolver {
 public:
  FullTreeSolver(const liars_dice::RecursiveSolvingParams& cfg, int device, int max_depth) {
    cfrb_config c = liars_dice::solver_config(cfg, device, 1);
    c.max_depth = max_depth;
    c.net_mode = CFRB_NET_ZERO;
    h_ = open_handle(c);
    A_ = cfrb_num_actions(h_.get()); H_ = cfrb_num_hands(h_.get()); N_ = cfrb_max_nodes(h_.get());
    std::vector<cfrb_node> t(N_);
    cfrb_tree_template(h_.get(), -1, 0, t.data(), N_);
    for (const auto& n : t)
      if (n.children_begin == n.children_end && n.last_bid != A_ - 1)   // subgame_solving.cc:181-184
        throw std::runtime_error("Found a non-final leaf node, but value_net is not provided");
    const int32_t lb = -1, pl = 0;
    std::vector<double> b((size_t)2 * H_, 1.0 / H_);
    check(cfrb_begin_wave(h_.get(), 1, &lb, &pl, b.data(), nullptr), "cfrb_begin_wave");
  }

  void step(int iters) { check(cfrb_run(h_.get(), iters, nullptr), "cfrb_run"); }
  std::vector<double> strategy() {   // get_strategy(): dense [N][H][A]
    std::vector<double> s((size_t)N_ * H_ * A_);
    check(cfrb_fetch(h_.get(), nullptr, nullptr, nullptr, s.data(), nullptr, nullptr), "cfrb_fetch");
    return s;
  }
  std::array<double, 2> exploitability(const std::vector<double>& s) {
    std::array<double, 2> e{};
    check(cfrb_exploitability(h_.get(), s.data(), e.data()), "cfrb_exploitability");
    return e;
  }
  cfrb_handle* handle() const { return h_.get(); }
  int numNodes() const { return N_; }

 private:
  HandlePtr h_;
  int A_ = 0, H_ = 0, N_ = 0;
};

// reach_probabilities[p][node][hand] from uniform beliefs and node_reach (compute_stategy_stats, subgame_solving.cc:823-846).
struct StrategyReach {
  std::vector<double> reach[2];   // [N][H]
  std::vector<double> node_reach; // [N]
};
inline StrategyReach strategy_reach(const std::vector<cfrb_node>& tree, int H, int A, const std::vector<double>& strategy) {
  const int N = (int)tree.size();
  StrategyReach r;
  for (int p = 0; p < 2; ++p) {
    r.reach[p].assign((size_t)N * H, 0.0);
    for (int n = 0; n < N; ++n)
      for (int h = 0; h < H; ++h) {
        if (n == 0) { r.reach[p][h] = 1.0 / H; continue; }
        const int par = tree[n].parent;
        const double rp = r.reach[p][(size_t)par * H + h];
        r.reach[p][(size_t)n * H + h] = tree[par].player_id == p ? rp * strategy[((size_t)par * H + h) * A + tree[n].last_bid] : rp;
      }
  }
  r.node_reach.resize(N);
  for (int n = N; n-- > 0;) {
    double s0 = 0, s1 = 0;
    for (int h = 0; h < H; ++h) { s0 += r.reach[0][(size_t)n * H + h]; s1 += r.reach[1][(size_t)n * H + h]; }
    r.node_reach[n] = s0 * s1;
  }
  return r;
}

// eval_net's candidates (stats.cc:64-72): the non-terminal nodes at depth mdp_depth and 2 * mdp_depth in node order, with their
// reach statistics under the net strategy ([0]) and the full-tree strategy ([1]): node_reach per candidate and both players'
// reach rows [candidate][2][H].
struct EvalNetCandidates {
  std::vector<int> node;
  std::vector<double> node_reach[2];
  std::vector<double> rows[2];
};
inline std::vector<int> eval_net_candidate_nodes(const std::vector<cfrb_node>& tree, int A, int mdp_depth) {
  std::vector<int> c;
  for (int i = 0; i < (int)tree.size(); ++i)
    if ((tree[i].depth == mdp_depth || tree[i].depth == 2 * mdp_depth) && tree[i].last_bid != A - 1) c.push_back(i);
  return c;
}

// root_value_means [n][2][H] of full-depth linear fictitious-play solves without a value net (stats.cc:118-124), the i-th rooted
// at nodes[i] with beliefs bel [i][2][H], iteration count params.subgame_params.num_iters.
using RootSolve = std::function<std::vector<double>(const std::vector<int>& nodes, const std::vector<double>& bel)>;

// eval_net (stats.cc:44-153): mean squared difference between the value net's prediction and a full-depth fictitious-play
// solve at the candidates reached with probability >= 1e-6 under the strategy that defines the beliefs.  Where the reach
// statistics and the root solves come from is the caller's; the selection, the queries, the forward and the MSE are here.
inline float eval_net_scored(const liars_dice::RecursiveSolvingParams& cfg, const std::vector<cfrb_node>& tree, const EvalNetCandidates& cand,
                             torch::jit::Module& model, bool traverse_by_net, bool verbose, const RootSolve& solve) {
  const int D = cfg.num_dice, F = cfg.num_faces, A = 1 + 2 * D * F;
  int H = 1;
  for (int i = 0; i < D; ++i) H *= F;
  const int Q = 2 + A + 2 * H;
  const int tv = traverse_by_net ? 0 : 1;
  const auto& node_reach = cand.node_reach[tv];
  std::vector<int> top(cand.node.size());   // candidate indices, in node order
  std::iota(top.begin(), top.end(), 0);
  std::sort(top.begin(), top.end(), [&node_reach](int i, int j) { return node_reach[i] > node_reach[j]; });
  const float kMinReach = 1e-6;
  if (top.empty()) return 0.0f;
  while (!top.empty() && node_reach[top.back()] < kMinReach) top.pop_back();
  if (top.empty()) return 0.0f;
  if (verbose)
    std::printf("eval_net (%s policy defines the beliefs): %zu nodes, reach %.3e .. %.3e\n", traverse_by_net ? "net" : "full-tree",
                top.size(), node_reach[top.back()], node_reach[top.front()]);

  const size_t n_top = top.size();
  std::vector<int> nodes(n_top);
  std::vector<double> bel(n_top * 2 * H);
  for (size_t i = 0; i < n_top; ++i) {
    nodes[i] = cand.node[top[i]];
    for (int p = 0; p < 2; ++p) {   // normalize_probabilities (util.h:20-34)
      const double* r = &cand.rows[tv][((size_t)top[i] * 2 + p) * H];
      double s = 0;
      for (int hh = 0; hh < H; ++hh) s += r[hh];
      for (int hh = 0; hh < H; ++hh) bel[(i * 2 + p) * H + hh] = r[hh] / s;
    }
  }
  const std::vector<double> mu = solve(nodes, bel);
  const int chunk = 64;
  std::vector<float> mses;
  for (size_t off = 0; off < n_top; off += chunk) {
    const int n = (int)std::min<size_t>(chunk, n_top - off);
    // net predictions for the 2n (node, traverser) queries of the chunk in ONE forward (the reference evaluates them one
    // row at a time, stats.cc:128-133; a [1,Q] forward per row costs milliseconds of thread wake-ups on a many-core host)
    std::vector<float> q((size_t)2 * n * Q, 0.f);
    for (int i = 0; i < n; ++i) {
      const int node = nodes[off + i];
      for (int t = 0; t < 2; ++t) {   // get_query / write_query_to (subgame_solving.cc:104-123,901-908)
        float* row = &q[((size_t)i * 2 + t) * Q];
        row[0] = (float)tree[node].player_id; row[1] = (float)t;
        if (tree[node].last_bid >= 0) row[2 + tree[node].last_bid] = 1.f;
        for (int p = 0; p < 2; ++p) {
          const double* b = &bel[((off + i) * 2 + p) * H];
          double s = 0;
          for (int hh = 0; hh < H; ++hh) s += b[hh] + 1e-80;
          for (int hh = 0; hh < H; ++hh) row[2 + A + p * H + hh] = (float)((b[hh] + 1e-80) / s);
        }
      }
    }
    torch::NoGradGuard ng;
    const auto net_out = model.forward({torch::from_blob(q.data(), {2 * n, Q}, torch::kFloat32).clone()}).toTensor().contiguous();
    for (int i = 0; i < n; ++i) {
      const int node = nodes[off + i], c = top[off + i];
      for (int t = 0; t < 2; ++t) {
        auto reach_t = torch::from_blob(const_cast<double*>(&bel[((off + i) * 2 + t) * H]), {H}, torch::kFloat64).clone();
        const float net_value = (net_out[i * 2 + t] * reach_t).sum().item<float>();
        auto hv = torch::from_blob(const_cast<double*>(&mu[((off + i) * 2 + t) * H]), {H}, torch::kFloat64).clone();
        const float br_value = (hv * reach_t).sum().item<float>();
        if (verbose)
          std::printf("  node %d (bid %d, player %d) traverser %d: net_reach=%.3e true_reach=%.3e net_value=%.5f br_value=%.5f\n", node,
                      tree[node].last_bid, tree[node].player_id, t, cand.node_reach[0][c], cand.node_reach[1][c], net_value, br_value);
        mses.push_back((float)std::pow(net_value - br_value, 2.0));
      }
    }
  }
  const float mse = std::accumulate(mses.begin(), mses.end(), 0.0f) / mses.size();
  if (verbose) std::printf("Final MSE: %g\n", mse);
  return mse;
}

// eval_net on dense strategies [N][H][A]: the reach statistics of strategy_reach, and the root solves as subgames of a wave handle
// (linear FP, max_depth 10000, no value net), 64 per wave.
inline float eval_net(const liars_dice::RecursiveSolvingParams& cfg, int device, const std::vector<cfrb_node>& tree,
                      const std::vector<double>& net_strategy, const std::vector<double>& full_strategy, torch::jit::Module& model,
                      bool traverse_by_net, bool verbose) {
  const int D = cfg.num_dice, F = cfg.num_faces, A = 1 + 2 * D * F;
  int H = 1;
  for (int i = 0; i < D; ++i) H *= F;
  const int fp_iters = cfg.subgame_params.num_iters;
  const StrategyReach stats[2] = {strategy_reach(tree, H, A, net_strategy), strategy_reach(tree, H, A, full_strategy)};
  EvalNetCandidates cand;
  cand.node = eval_net_candidate_nodes(tree, A, cfg.subgame_params.max_depth);
  for (int s = 0; s < 2; ++s)
    for (int node : cand.node) {
      cand.node_reach[s].push_back(stats[s].node_reach[node]);
      for (int p = 0; p < 2; ++p)
        cand.rows[s].insert(cand.rows[s].end(), &stats[s].reach[p][(size_t)node * H], &stats[s].reach[p][(size_t)(node + 1) * H]);
    }
  auto solve = [&](const std::vector<int>& nodes, const std::vector<double>& bel) {
    liars_dice::RecursiveSolvingParams fpc = cfg;
    fpc.subgame_params = liars_dice::SubgameSolvingParams();     // defaults: FP
    fpc.subgame_params.linear_update = true;
    fpc.subgame_params.max_depth = 10000;
    fpc.subgame_params.num_iters = fp_iters;
    fpc.net_mode = CFRB_NET_ZERO;
    const int chunk = 64;
    const HandlePtr h = open_handle(liars_dice::solver_config(fpc, device, chunk));
    std::vector<double> mu(bel.size());
    for (size_t off = 0; off < nodes.size(); off += chunk) {
      const int n = (int)std::min<size_t>(chunk, nodes.size() - off);
      std::vector<int32_t> lb(n), pl(n);
      for (int i = 0; i < n; ++i) { lb[i] = tree[nodes[off + i]].last_bid; pl[i] = tree[nodes[off + i]].player_id; }
      check(cfrb_begin_wave(h.get(), n, lb.data(), pl.data(), &bel[off * 2 * H], nullptr), "cfrb_begin_wave");
      check(cfrb_run(h.get(), fp_iters, nullptr), "cfrb_run");
      check(cfrb_fetch(h.get(), &mu[off * 2 * H], nullptr, nullptr, nullptr, nullptr, nullptr), "cfrb_fetch");
    }
    return mu;
  };
  return eval_net_scored(cfg, tree, cand, model, traverse_by_net, verbose, solve);
}

using FpForestPtr = std::unique_ptr<cfrb_fp_forest, Destroyer<cfrb_fp_forest_destroy>>;

// eval_net's candidates with the reach statistics of two compact full-tree strategies [N - 1][H], formed on the device
// (cfrb_fp_forest_reach): the same bits as strategy_reach's.
inline EvalNetCandidates forest_candidates(cfrb_fp_forest* f, const std::vector<cfrb_node>& tree, int A, int H, int mdp_depth,
                                           const std::vector<double>& net_compact, const std::vector<double>& full_compact) {
  EvalNetCandidates cand;
  cand.node = eval_net_candidate_nodes(tree, A, mdp_depth);
  if (cand.node.empty()) return cand;
  const int n = (int)cand.node.size();
  const std::vector<double>* s[2] = {&net_compact, &full_compact};
  for (int k = 0; k < 2; ++k) {
    cand.node_reach[k].resize(n);
    cand.rows[k].resize((size_t)n * 2 * H);
    check(cfrb_fp_forest_reach(f, s[k]->data(), n, cand.node.data(), cand.node_reach[k].data(), cand.rows[k].data()),
          "cfrb_fp_forest_reach");
  }
  return cand;
}

// eval_net's root solves on the device: one forest solve per depth over the roots of that depth (cfrb_fp_forest_solve, the bits
// of the wave subgames above).  after(depth, roots) is called after each depth's solve.
inline RootSolve forest_root_solve(cfrb_fp_forest* f, const std::vector<cfrb_node>& tree, int H, int iters,
                                   std::function<void(int, size_t)> after = nullptr) {
  return [f, &tree, H, iters, after](const std::vector<int>& nodes, const std::vector<double>& bel) {
    std::vector<double> mu(bel.size());
    std::vector<int> depths;
    for (int v : nodes) depths.push_back(tree[v].depth);
    std::sort(depths.begin(), depths.end());
    depths.erase(std::unique(depths.begin(), depths.end()), depths.end());
    for (int d : depths) {
      std::vector<int> idx;   // positions of this depth's roots, by node id (the forest takes them ascending)
      for (size_t i = 0; i < nodes.size(); ++i)
        if (tree[nodes[i]].depth == d) idx.push_back((int)i);
      std::sort(idx.begin(), idx.end(), [&](int a, int b) { return nodes[a] < nodes[b]; });
      std::vector<int32_t> roots;
      std::vector<double> b, m(idx.size() * 2 * H);
      for (int i : idx) {
        roots.push_back(nodes[i]);
        b.insert(b.end(), &bel[(size_t)i * 2 * H], &bel[(size_t)(i + 1) * 2 * H]);
      }
      check(cfrb_fp_forest_solve(f, d, (int)roots.size(), roots.data(), b.data(), iters, m.data()), "cfrb_fp_forest_solve");
      for (size_t k = 0; k < idx.size(); ++k) std::copy(&m[k * 2 * H], &m[(k + 1) * 2 * H], &mu[(size_t)idx[k] * 2 * H]);
      if (after) after(d, roots.size());
    }
    return mu;
  };
}

}  // namespace rela
