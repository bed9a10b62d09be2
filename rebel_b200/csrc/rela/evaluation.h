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
#include <memory>
#include <numeric>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "../../../include/cfrb200.h"
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
    const auto& sp = cfg.subgame_params;
    cfrb_config c{};
    c.num_dice = cfg.num_dice; c.num_faces = cfg.num_faces; c.max_depth = max_depth; c.num_iters = sp.num_iters;
    c.linear_update = sp.linear_update; c.dcfr = sp.dcfr; c.dcfr_alpha = sp.dcfr_alpha; c.dcfr_beta = sp.dcfr_beta;
    c.dcfr_gamma = sp.dcfr_gamma; c.max_subgames = 1; c.device = device; c.net_mode = CFRB_NET_ZERO; c.hidden = 256;
    c.state_dtype = cfg.state_dtype;
    c.solver = sp.use_cfr ? CFRB_SOLVER_CFR : CFRB_SOLVER_FP;
    c.optimistic = sp.optimistic;
    if (cfrb_create(&c, &h_) < 0) throw std::runtime_error(std::string("cfrb_create: ") + cfrb_last_error());
    A_ = cfrb_num_actions(h_); H_ = cfrb_num_hands(h_); N_ = cfrb_max_nodes(h_);
    std::vector<cfrb_node> t(N_);
    cfrb_tree_template(h_, -1, 0, t.data(), N_);
    for (const auto& n : t)
      if (n.children_begin == n.children_end && n.last_bid != A_ - 1)   // subgame_solving.cc:181-184
        throw std::runtime_error("Found a non-final leaf node, but value_net is not provided");
    const int32_t lb = -1, pl = 0;
    std::vector<double> b((size_t)2 * H_, 1.0 / H_);
    if (cfrb_begin_wave(h_, 1, &lb, &pl, b.data(), nullptr) < 0) throw std::runtime_error(cfrb_last_error());
  }
  ~FullTreeSolver() { if (h_) cfrb_destroy(h_); }
  FullTreeSolver(const FullTreeSolver&) = delete;
  FullTreeSolver& operator=(const FullTreeSolver&) = delete;

  void step(int iters) { if (cfrb_run(h_, iters, nullptr) < 0) throw std::runtime_error(cfrb_last_error()); }
  std::vector<double> strategy() {   // get_strategy(): dense [N][H][A]
    std::vector<double> s((size_t)N_ * H_ * A_);
    if (cfrb_fetch(h_, nullptr, nullptr, nullptr, s.data(), nullptr, nullptr) < 0) throw std::runtime_error(cfrb_last_error());
    return s;
  }
  std::array<double, 2> exploitability(const std::vector<double>& s) {
    std::array<double, 2> e{};
    if (cfrb_exploitability(h_, s.data(), e.data()) < 0) throw std::runtime_error(cfrb_last_error());
    return e;
  }
  cfrb_handle* handle() const { return h_; }
  int numNodes() const { return N_; }

 private:
  cfrb_handle* h_ = nullptr;
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

// eval_net (stats.cc:44-153): mean squared difference between the value net's prediction and a full-depth fictitious-play
// solve at the non-terminal nodes of depth mdp_depth and 2*mdp_depth reached with probability >= 1e-6.
inline float eval_net(const liars_dice::RecursiveSolvingParams& cfg, int device, const std::vector<cfrb_node>& tree,
                      const std::vector<double>& net_strategy, const std::vector<double>& full_strategy, torch::jit::Module& model,
                      bool traverse_by_net, bool verbose) {
  const int D = cfg.num_dice, F = cfg.num_faces, A = 1 + 2 * D * F;
  int H = 1;
  for (int i = 0; i < D; ++i) H *= F;
  const int Q = 2 + A + 2 * H, mdp_depth = cfg.subgame_params.max_depth, fp_iters = cfg.subgame_params.num_iters;
  const StrategyReach net_stats = strategy_reach(tree, H, A, net_strategy), true_stats = strategy_reach(tree, H, A, full_strategy);
  const StrategyReach& trav = traverse_by_net ? net_stats : true_stats;
  std::vector<int> top;
  for (int i = 0; i < (int)tree.size(); ++i)
    if ((tree[i].depth == mdp_depth || tree[i].depth == 2 * mdp_depth) && tree[i].last_bid != A - 1) top.push_back(i);
  const auto& node_reach = trav.node_reach;
  std::sort(top.begin(), top.end(), [&node_reach](int i, int j) { return node_reach[i] > node_reach[j]; });
  const float kMinReach = 1e-6;
  if (top.empty()) return 0.0f;
  while (!top.empty() && node_reach[top.back()] < kMinReach) top.pop_back();
  if (top.empty()) return 0.0f;
  if (verbose)
    std::printf("eval_net (%s policy defines the beliefs): %zu nodes, reach %.3e .. %.3e\n", traverse_by_net ? "net" : "full-tree",
                top.size(), node_reach[top.back()], node_reach[top.front()]);

  // full-depth linear fictitious play from every selected node (stats.cc:118-124), one wave per chunk
  liars_dice::RecursiveSolvingParams fpc = cfg;
  fpc.subgame_params = liars_dice::SubgameSolvingParams();     // defaults: FP, max_depth irrelevant here
  const int chunk = 64;
  cfrb_config c{};
  c.num_dice = D; c.num_faces = F; c.max_depth = 10000; c.num_iters = fp_iters; c.linear_update = 1; c.max_subgames = chunk;
  c.device = device; c.net_mode = CFRB_NET_ZERO; c.hidden = 256; c.state_dtype = cfg.state_dtype; c.solver = CFRB_SOLVER_FP;
  cfrb_handle* h = nullptr;
  if (cfrb_create(&c, &h) < 0) throw std::runtime_error(std::string("cfrb_create: ") + cfrb_last_error());
  std::vector<float> mses;
  try {
    for (size_t off = 0; off < top.size(); off += chunk) {
      const int n = (int)std::min<size_t>(chunk, top.size() - off);
      std::vector<int32_t> lb(n), pl(n);
      std::vector<double> bel((size_t)n * 2 * H), mu((size_t)n * 2 * H);
      for (int i = 0; i < n; ++i) {
        const int node = top[off + i];
        lb[i] = tree[node].last_bid; pl[i] = tree[node].player_id;
        for (int p = 0; p < 2; ++p) {   // normalize_probabilities (util.h:20-34)
          const double* r = &trav.reach[p][(size_t)node * H];
          double s = 0;
          for (int hh = 0; hh < H; ++hh) s += r[hh];
          for (int hh = 0; hh < H; ++hh) bel[((size_t)i * 2 + p) * H + hh] = r[hh] / s;
        }
      }
      if (cfrb_begin_wave(h, n, lb.data(), pl.data(), bel.data(), nullptr) < 0) throw std::runtime_error(cfrb_last_error());
      if (cfrb_run(h, fp_iters, nullptr) < 0) throw std::runtime_error(cfrb_last_error());
      if (cfrb_fetch(h, mu.data(), nullptr, nullptr, nullptr, nullptr, nullptr) < 0) throw std::runtime_error(cfrb_last_error());
      // net predictions for the 2n (node, traverser) queries of the chunk in ONE forward (the reference evaluates them one
      // row at a time, stats.cc:128-133; a [1,Q] forward per row costs milliseconds of thread wake-ups on a many-core host)
      std::vector<float> q((size_t)2 * n * Q, 0.f);
      for (int i = 0; i < n; ++i) {
        const int node = top[off + i];
        for (int t = 0; t < 2; ++t) {   // get_query / write_query_to (subgame_solving.cc:104-123,901-908)
          float* row = &q[((size_t)i * 2 + t) * Q];
          row[0] = (float)tree[node].player_id; row[1] = (float)t;
          if (tree[node].last_bid >= 0) row[2 + tree[node].last_bid] = 1.f;
          for (int p = 0; p < 2; ++p) {
            const double* b = &bel[((size_t)i * 2 + p) * H];
            double s = 0;
            for (int hh = 0; hh < H; ++hh) s += b[hh] + 1e-80;
            for (int hh = 0; hh < H; ++hh) row[2 + A + p * H + hh] = (float)((b[hh] + 1e-80) / s);
          }
        }
      }
      torch::NoGradGuard ng;
      const auto net_out = model.forward({torch::from_blob(q.data(), {2 * n, Q}, torch::kFloat32).clone()}).toTensor().contiguous();
      for (int i = 0; i < n; ++i) {
        const int node = top[off + i];
        for (int t = 0; t < 2; ++t) {
          auto reach_t = torch::from_blob(&bel[((size_t)i * 2 + t) * H], {H}, torch::kFloat64).clone();
          const float net_value = (net_out[i * 2 + t] * reach_t).sum().item<float>();
          auto hv = torch::from_blob(&mu[((size_t)i * 2 + t) * H], {H}, torch::kFloat64).clone();
          const float br_value = (hv * reach_t).sum().item<float>();
          if (verbose)
            std::printf("  node %d (bid %d, player %d) traverser %d: net_reach=%.3e true_reach=%.3e net_value=%.5f br_value=%.5f\n", node,
                        tree[node].last_bid, tree[node].player_id, t, net_stats.node_reach[node], true_stats.node_reach[node], net_value,
                        br_value);
          mses.push_back((float)std::pow(net_value - br_value, 2.0));
        }
      }
    }
  } catch (...) {
    cfrb_destroy(h);
    throw;
  }
  cfrb_destroy(h);
  const float mse = std::accumulate(mses.begin(), mses.end(), 0.0f) / mses.size();
  if (verbose) std::printf("Final MSE: %g\n", mse);
  return mse;
}

}  // namespace rela
