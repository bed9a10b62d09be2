// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// Thin extern "C" harness around the UNMODIFIED reference sources compiled where they
// lie in a checkout of the original project (recipe: oracle/Makefile, output: oracle/_ref/).  It exists so
// that (1) the plain-C restatement in oracle/cfr_oracle.c can be pinned against the real
// reference, (2) golden fixtures under tests/golden/ can be generated (oracle/make_golden.py)
// and (3) bench.py's `--impl reference` / `cpu_baseline` leg can time the reference's own
// CPU implementation of the hot path on the host cores.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
// may load the resulting library.  Nothing in rebel_b200/ links or dlopens it.
//
// The CFR solver class lives in an anonymous namespace of subgame_solving.cc
// (subgame_solving.cc:508-715) with private state, so this TU #includes that .cc file
// verbatim (no copy is made) with private/protected opened up to be able to dump
// regrets / sum_strategies / leaf values for teacher-forced parity tests.

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <memory>
#include <mutex>
#include <numeric>
#include <queue>
#include <random>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include <torch/script.h>
#include <torch/torch.h>

#define private public
#define protected public
#include "subgame_solving.cc"  // reference source, found through -I$(REF)/csrc/liars_dice
#undef private
#undef protected

#include "real_net.h"
#include "recursive_solving.h"
#include "stats.h"

using namespace liars_dice;

namespace {

thread_local std::string g_err;
thread_local double g_noise_rel = 0;       // ref_set_net_noise: relative gaussian noise on the Net2 outputs of ref_cfr_solve
thread_local uint64_t g_noise_seed = 0;
thread_local int g_net_emulation = 0;      // ref_set_net_emulation: 0 fp32 ATen (the reference), 1 / 2 arithmetic model of the tensor-core kernels

SubgameSolvingParams make_params(int num_iters, int max_depth, int linear_update, int dcfr,
                                 double dcfr_alpha, double dcfr_beta, double dcfr_gamma) {
  SubgameSolvingParams p;
  p.num_iters = num_iters;
  p.max_depth = max_depth;
  p.linear_update = linear_update != 0;
  p.use_cfr = true;
  p.dcfr = dcfr != 0;
  p.dcfr_alpha = dcfr_alpha;
  p.dcfr_beta = dcfr_beta;
  p.dcfr_gamma = dcfr_gamma;
  return p;
}

// Value net that evaluates Net2 (models.py:64-94) with ATen CPU ops from a flat fp32
// weight buffer in state_dict order.  Same ATen kernels the TorchScript module dispatches to.
class FlatNet2 : public IValueNet {
 public:
  FlatNet2(const float* w, int Q, int hidden, int H) {
    auto take = [&](std::vector<int64_t> shape) {
      int64_t n = 1;
      for (auto s : shape) n *= s;
      auto t = torch::from_blob(const_cast<float*>(w), shape, torch::kFloat32).clone();
      w += n;
      return t;
    };
    w1 = take({hidden, Q}); b1 = take({hidden}); g1 = take({hidden}); be1 = take({hidden});
    w2 = take({hidden, hidden}); b2 = take({hidden}); g2 = take({hidden}); be2 = take({hidden});
    w3 = take({H, hidden}); b3 = take({H});
    hidden_ = hidden;
  }
  // Arithmetic model of the tensor-core value-net kernels (rebel_b200/csrc/leaf_mlp_tc.cuh) inside the reference's own net, used
  // to derive parity bands (make_golden_r2.py): query columns, weights and both hidden activations rounded to fp16 (fp32
  // accumulation, fp32 LayerNorm), GELU either in fp32 (model 1, CFRB_NET_TC_F16: the 3-term logistic form) or in packed-half
  // arithmetic with one rounding per HMUL2 / HFMA2 / tanh (model 2, CFRB_NET_TC_F16X2).
  static torch::Tensor h16(const torch::Tensor& x) { return x.to(torch::kHalf).to(torch::kFloat32); }   // one fp16 rounding
  static torch::Tensor gelu_model(const torch::Tensor& y, int model) {
    if (model == 1) {      // gelu_tc (leaf_mlp_tc.cuh): y / (1 + 2^(y p(y^2))) in fp32, result rounded to fp16
      auto y2 = (y * y).clamp_max(52.f);
      auto p = y2 * (y2 * 1.014244e-3f - 1.0677588e-1f) - 2.3011216f;
      return h16(y / (1.f + torch::exp2(y * p)));
    }
    // gelu_hy_x2 (leaf_mlp_tc.cuh): hy = y / 2 rounded to fp16, then HMUL2 / HFMA2 / tanh.approx.f16x2 with one rounding each
    // (the fp32 product of two fp16 values is exact, so rounding the fp32 result of a*b+c once models the fused HFMA2)
    const float c2 = (float)(at::Half)(-1.124832e-2f), c1 = (float)(at::Half)(2.960456e-1f), c0 = (float)(at::Half)(1.594992f);
    auto hy = h16(0.5f * y);
    auto s = h16(hy * hy).clamp_max(13.f);
    auto p = h16(s * h16(s * c2 + c1) + c0);
    auto u = h16(hy * p);
    auto t = h16(torch::tanh(u));
    return h16(hy * t + hy);
  }
  torch::Tensor hidden_model(torch::Tensor pre, const torch::Tensor& g, const torch::Tensor& be, int model) {
    return gelu_model(torch::layer_norm(pre, {hidden_}, g, be, 1e-5), model);
  }
  torch::Tensor compute_values(const torch::Tensor q) override {
    torch::NoGradGuard ng;
    torch::Tensor y;
    if (emulation) {
      if (!w1h.defined()) { w1h = w1.to(torch::kHalf).to(torch::kFloat32); w2h = w2.to(torch::kHalf).to(torch::kFloat32); w3h = w3.to(torch::kHalf).to(torch::kFloat32); }
      auto x = hidden_model(torch::linear(q.to(torch::kHalf).to(torch::kFloat32), w1h, b1), g1, be1, emulation);
      x = hidden_model(torch::linear(x, w2h, b2), g2, be2, emulation);
      y = torch::linear(x, w3h, b3);
    } else {
      auto x = torch::gelu(torch::layer_norm(torch::linear(q, w1, b1), {hidden_}, g1, be1, 1e-5));
      x = torch::gelu(torch::layer_norm(torch::linear(x, w2, b2), {hidden_}, g2, be2, 1e-5));
      y = torch::linear(x, w3, b3);
    }
    if (noise_rel > 0) {   // parity-band experiments (SURVEY appendix B "pert"): outputs * (1 + rel * N(0,1)), seeded
      float* p = y.data_ptr<float>();
      std::normal_distribution<double> n01(0.0, 1.0);
      for (int64_t i = 0; i < y.numel(); ++i) p[i] = (float)(p[i] * (1.0 + noise_rel * n01(noise_gen)));
    }
    return y;
  }
  int emulation = 0;
  torch::Tensor w1h, w2h, w3h;
  double noise_rel = 0;
  std::mt19937_64 noise_gen{0};
  void add_training_example(const torch::Tensor q, const torch::Tensor v) override {
    std::lock_guard<std::mutex> lk(m_);
    const float* qp = q.data_ptr<float>();
    const float* vp = v.data_ptr<float>();
    examples_q.insert(examples_q.end(), qp, qp + q.numel());
    examples_v.insert(examples_v.end(), vp, vp + v.numel());
    ++n_examples;
  }
  std::vector<float> examples_q, examples_v;
  std::atomic<int64_t> n_examples{0};

 private:
  torch::Tensor w1, b1, g1, be1, w2, b2, g2, be2, w3, b3;
  int64_t hidden_;
  std::mutex m_;
};

// Zero net that records the training examples (real_net.cc:30-55 drops them).
class RecordingZeroNet : public IValueNet {
 public:
  explicit RecordingZeroNet(int H) : H_(H) {}
  torch::Tensor compute_values(const torch::Tensor q) override {
    return torch::zeros({q.size(0), H_});
  }
  void add_training_example(const torch::Tensor q, const torch::Tensor v) override {
    std::lock_guard<std::mutex> lk(m_);
    const float* qp = q.data_ptr<float>();
    const float* vp = v.data_ptr<float>();
    examples_q.insert(examples_q.end(), qp, qp + q.numel());
    examples_v.insert(examples_v.end(), vp, vp + v.numel());
  }
  std::vector<float> examples_q, examples_v;

 private:
  int64_t H_;
  std::mutex m_;
};

// TorchScript net on CPU that also counts examples (for the timed baseline: identical code
// path to rela::ModelLocker::forward on device "cpu", model_locker.h:85-95).
class CountingScriptNet : public IValueNet {
 public:
  explicit CountingScriptNet(const std::string& path) : module_(torch::jit::load(path)) {
    module_.eval();
  }
  torch::Tensor compute_values(const torch::Tensor q) override {
    torch::NoGradGuard ng;
    std::vector<torch::jit::IValue> in = {q};
    return torch::detach(module_.forward(in).toTensor());
  }
  void add_training_example(const torch::Tensor, const torch::Tensor) override { ++n_examples; }
  std::atomic<int64_t> n_examples{0};

 private:
  torch::jit::script::Module module_;
};

void dump_dense(const TreeStrategy& s, double* out) {
  if (!out) return;
  size_t k = 0;
  for (auto& n : s)
    for (auto& h : n)
      for (double v : h) out[k++] = v;
}

Pair<std::vector<double>> to_beliefs(const double* b, int H) {
  Pair<std::vector<double>> beliefs;
  beliefs[0].assign(b, b + H);
  beliefs[1].assign(b + H, b + 2 * H);
  return beliefs;
}

}  // namespace

extern "C" {

const char* ref_last_error() { return g_err.c_str(); }

// Parity-band experiments: the next ref_cfr_solve calls of this thread multiply every value-net output by 1 + rel * N(0,1).
void ref_set_net_noise(double rel, uint64_t seed) { g_noise_rel = rel; g_noise_seed = seed; }
void ref_set_net_emulation(int model) { g_net_emulation = model; }

// tree.h:51-70.  out rows: last_bid, player_id, children_begin, children_end, parent, depth.
int ref_unroll_tree(int D, int F, int last_bid, int player_id, int max_depth, int32_t* out,
                    int cap_nodes) {
  Game game(D, F);
  PartialPublicState root{last_bid, player_id};
  auto tree = unroll_tree(game, root, max_depth);
  if ((int)tree.size() > cap_nodes) return -(int)tree.size();
  for (size_t i = 0; i < tree.size(); ++i) {
    int32_t* r = out + 6 * i;
    r[0] = tree[i].state.last_bid;
    r[1] = tree[i].state.player_id;
    r[2] = tree[i].children_begin;
    r[3] = tree[i].children_end;
    r[4] = tree[i].parent;
    r[5] = tree[i].depth;
  }
  return (int)tree.size();
}

int ref_num_matches(int D, int F, int hand, int face) { return Game(D, F).num_matches(hand, face); }

// subgame_solving.cc:765-789
void ref_win_probability(int D, int F, int bet, const double* beliefs, double* out) {
  Game game(D, F);
  std::vector<double> b(beliefs, beliefs + game.num_hands());
  auto v = compute_win_probability(game, bet, b);
  std::copy(v.begin(), v.end(), out);
}

// subgame_solving.cc:104-123 via get_query
int ref_query(int D, int F, int traverser, int last_bid, int player_id, const double* r0,
              const double* r1, float* out) {
  Game game(D, F);
  std::vector<double> a(r0, r0 + game.num_hands()), b(r1, r1 + game.num_hands());
  auto q = get_query(game, traverser, PartialPublicState{last_bid, player_id}, a, b);
  std::copy(q.begin(), q.end(), out);
  return (int)q.size();
}

// Runs CFR (subgame_solving.cc:508-715) on one subgame and dumps the complete solver state at the
// requested checkpoints.  net_w == nullptr -> zero net if the tree has pseudo-leaves, else no net.
// Dense dumps are [N][H][A] doubles.  checkpoints[] are iteration counts (state AFTER that many
// steps), increasing.  leaf_values_out (optional) receives, for every checkpoint c>0, the
// [L][H] float leaf values (already multiplied by the scaler) that step c-1 consumed, and
// queries_out the [L][Q] float query rows of that step.
int ref_cfr_solve(int D, int F, int last_bid, int player_id, const double* beliefs, int num_iters,
                  int max_depth, int linear_update, int dcfr, double dcfr_alpha, double dcfr_beta,
                  double dcfr_gamma, const float* net_w, int hidden, int n_checkpoints,
                  const int32_t* checkpoints, double* regrets, double* last, double* sum,
                  double* avg, double* root_means /*[C][2][H]*/, float* leaf_values_out,
                  float* queries_out, double* traverser_values_out /*[C][N][H]*/) {
  try {
    Game game(D, F);
    const int H = game.num_hands(), A = game.num_actions();
    auto params = make_params(num_iters, max_depth, linear_update, dcfr, dcfr_alpha, dcfr_beta,
                              dcfr_gamma);
    PartialPublicState root{last_bid, player_id};
    auto tree = unroll_tree(game, root, max_depth);
    bool has_pleaf = false;
    for (auto& n : tree) has_pleaf |= (!n.num_children() && !game.is_terminal(n.state));
    std::shared_ptr<IValueNet> net;
    if (net_w) {
      auto n2 = std::make_shared<FlatNet2>(net_w, 2 + A + 2 * H, hidden, H);
      n2->noise_rel = g_noise_rel;
      n2->noise_gen.seed(g_noise_seed);
      n2->emulation = g_net_emulation;
      net = n2;
    } else if (has_pleaf) {
      net = create_zero_net(H, false);
    }
    CFR cfr(game, root, net, to_beliefs(beliefs, H), params);
    const size_t N = cfr.tree.size();
    const size_t dense = N * H * A;
    const size_t L = cfr.pseudo_leaves_indices.size();
    const size_t Q = cfr.query_size;
    int done = 0;
    for (int c = 0; c < n_checkpoints; ++c) {
      for (; done < checkpoints[c]; ++done) cfr.step(done % 2);
      dump_dense(cfr.regrets, regrets ? regrets + c * dense : nullptr);
      dump_dense(cfr.last_strategies, last ? last + c * dense : nullptr);
      dump_dense(cfr.sum_strategies, sum ? sum + c * dense : nullptr);
      dump_dense(cfr.average_strategies, avg ? avg + c * dense : nullptr);
      if (root_means) {
        for (int p = 0; p < 2; ++p)
          for (int h = 0; h < H; ++h)
            root_means[(c * 2 + p) * H + h] =
                (int)cfr.root_values_means[p].size() == H ? cfr.root_values_means[p][h] : 0.0;
      }
      if (leaf_values_out && L && done > 0) {
        auto lv = cfr.leaf_values.contiguous();
        std::memcpy(leaf_values_out + c * L * H, lv.data_ptr<float>(), L * H * sizeof(float));
      }
      if (queries_out && L && done > 0) {
        std::memcpy(queries_out + c * L * Q, cfr.net_query_buffer.data(), L * Q * sizeof(float));
      }
      if (traverser_values_out) {
        for (size_t n = 0; n < N; ++n)
          for (int h = 0; h < H; ++h)
            traverser_values_out[(c * N + n) * H + h] = cfr.traverser_values[n][h];
      }
    }
    return (int)N;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// The reference's other solver, fictitious play (FP, subgame_solving.cc:364-506): same dumps as ref_cfr_solve minus regrets.
int ref_fp_solve(int D, int F, int last_bid, int player_id, const double* beliefs, int num_iters, int max_depth,
                 int linear_update, int optimistic, const float* net_w, int hidden, int n_checkpoints,
                 const int32_t* checkpoints, double* last, double* sum, double* avg, double* root_means /*[C][2][H]*/) {
  try {
    Game game(D, F);
    const int H = game.num_hands(), A = game.num_actions();
    auto params = make_params(num_iters, max_depth, linear_update, 0, 0, 0, 0);
    params.use_cfr = false;
    params.optimistic = optimistic != 0;
    PartialPublicState root{last_bid, player_id};
    auto tree = unroll_tree(game, root, max_depth);
    bool has_pleaf = false;
    for (auto& n : tree) has_pleaf |= (!n.num_children() && !game.is_terminal(n.state));
    std::shared_ptr<IValueNet> net;
    if (net_w) {
      net = std::make_shared<FlatNet2>(net_w, 2 + A + 2 * H, hidden, H);
    } else if (has_pleaf) {
      net = create_zero_net(H, false);
    }
    FP fp(game, root, net, to_beliefs(beliefs, H), params);
    const size_t N = fp.tree.size();
    const size_t dense = N * H * A;
    int done = 0;
    for (int c = 0; c < n_checkpoints; ++c) {
      for (; done < checkpoints[c]; ++done) fp.step(done % 2);
      dump_dense(fp.last_strategies, last ? last + c * dense : nullptr);
      dump_dense(fp.sum_strategies, sum ? sum + c * dense : nullptr);
      dump_dense(fp.average_strategies, avg ? avg + c * dense : nullptr);
      if (root_means) {
        for (int p = 0; p < 2; ++p)
          for (int h = 0; h < H; ++h)
            root_means[(c * 2 + p) * H + h] = (int)fp.root_values_means[p].size() == H ? fp.root_values_means[p][h] : 0.0;
      }
    }
    return (int)N;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// What the evaluation entry points of rela/pybind.cc:45-84 compute, with the Net2 weights given flat:
//   strategy_recursive / out[0]: compute_strategy_recursive + compute_exploitability      (compute_exploitability_with_net)
//   strategy_to_leaf / out[1..3]: compute_strategy_recursive_to_leaf + exploitability, eval_net with the net strategy and with
//                                 the full-tree strategy defining the beliefs                 (compute_stats_with_net)
int ref_net_evaluation(int D, int F, int num_iters, int max_depth, int linear_update, int use_cfr, const float* net_w, int hidden,
                       int what /*1 recursive, 2 stats, 3 both*/, double* strategy_recursive, double* strategy_to_leaf, double* out4) {
  try {
    Game game(D, F);
    const int H = game.num_hands(), A = game.num_actions();
    auto params = make_params(num_iters, max_depth, linear_update, 0, 0, 0, 0);
    params.use_cfr = use_cfr != 0;
    std::shared_ptr<IValueNet> net = std::make_shared<FlatNet2>(net_w, 2 + A + 2 * H, hidden, H);
    auto dump = [&](const TreeStrategy& s, double* out) {
      if (!out) return;
      size_t k = 0;
      for (auto& n : s) {
        if (n.empty()) { k += (size_t)H * A; continue; }
        for (auto& h : n) for (double v : h) out[k++] = v;
      }
    };
    if (what & 1) {
      const auto s = compute_strategy_recursive(game, params, net);
      dump(s, strategy_recursive);
      out4[0] = compute_exploitability(game, s);
    }
    if (what & 2) {
      const auto net_strategy = compute_strategy_recursive_to_leaf(game, params, net);
      dump(net_strategy, strategy_to_leaf);
      out4[1] = compute_exploitability(game, net_strategy);
      auto full_params = params;
      full_params.max_depth = 100000;
      auto fp = build_solver(game, full_params);
      fp->multistep();
      const auto& full_strategy = fp->get_strategy();
      out4[2] = eval_net(game, net_strategy, full_strategy, params.max_depth, params.num_iters, net, true, false);
      out4[3] = eval_net(game, net_strategy, full_strategy, params.max_depth, params.num_iters, net, false, false);
    }
    return (int)unroll_tree(game).size();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// Full-tree exploitability of a dense [N][H][A] strategy (subgame_solving.cc:802-816).
int ref_exploitability(int D, int F, const double* strategy, double* out2) {
  try {
    Game game(D, F);
    auto tree = unroll_tree(game);
    TreeStrategy s;
    init_nd(tree.size(), game.num_hands(), game.num_actions(), 0.0, &s);
    size_t k = 0;
    for (auto& n : s)
      for (auto& h : n)
        for (double& v : h) v = strategy[k++];
    auto e = compute_exploitability2(game, s);
    out2[0] = e[0];
    out2[1] = e[1];
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// Runs RlRunner::step (recursive_solving.cc:160-182) `n_games` times with seed, recording every training example.  net_w ==
// nullptr -> zero net.  use_cfr = false is the fictitious-play solver (SubgameSolvingParams::use_cfr = false, the YAML default).
// Same signature as orc_rl_runner; the subgame limit and the per-subgame trace are the port's alone (max_subgames must be 0 and
// trace null here).  Returns #examples, fills up to cap.
int ref_rl_runner(int D, int F, int num_iters, int max_depth, int linear_update, float random_action_prob, int sample_leaf, int seed,
                  int n_games, const float* net_w, int hidden, float* q_out, float* v_out, int cap, int use_cfr, int optimistic,
                  int dcfr, double dcfr_alpha, double dcfr_beta, double dcfr_gamma, int max_subgames, int32_t* trace,
                  int trace_cap) {
  (void)trace_cap;
  if (max_subgames != 0 || trace) {
    g_err = "ref_rl_runner: max_subgames and trace are not available in the reference build";
    return -1;
  }
  try {
    Game game(D, F);
    const int H = game.num_hands(), A = game.num_actions(), Q = 2 + A + 2 * H;
    RecursiveSolvingParams cfg;
    cfg.num_dice = D;
    cfg.num_faces = F;
    cfg.random_action_prob = random_action_prob;
    cfg.sample_leaf = sample_leaf != 0;
    cfg.subgame_params = make_params(num_iters, max_depth, linear_update, use_cfr ? dcfr : 0, dcfr_alpha, dcfr_beta, dcfr_gamma);
    cfg.subgame_params.use_cfr = use_cfr != 0;
    cfg.subgame_params.optimistic = optimistic != 0;
    std::vector<float>*eq, *ev;
    std::shared_ptr<IValueNet> net;
    if (net_w) {
      auto n = std::make_shared<FlatNet2>(net_w, Q, hidden, H);
      n->emulation = g_net_emulation;
      n->noise_rel = g_noise_rel;
      n->noise_gen.seed(g_noise_seed + (uint64_t)seed);
      eq = &n->examples_q;
      ev = &n->examples_v;
      net = n;
    } else {
      auto n = std::make_shared<RecordingZeroNet>(H);
      eq = &n->examples_q;
      ev = &n->examples_v;
      net = n;
    }
    RlRunner runner(cfg, net, seed);
    for (int g = 0; g < n_games; ++g) runner.step();
    int n = (int)(ev->size() / H);
    int m = std::min(n, cap);
    std::memcpy(q_out, eq->data(), sizeof(float) * m * Q);
    std::memcpy(v_out, ev->data(), sizeof(float) * m * H);
    return n;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// One sampled recursive strategy (BASELINE config 5 unit): compute_sampled_strategy_recursive_to_leaf
// (recursive_solving.cc:301-327).  net_w == nullptr -> zero net.  strategy_out: dense [N_full][H][A] doubles.
// Also returns, per full-tree node that roots a subgame, the sampled act_iteration (-1 elsewhere) by re-running the
// same mt19937 stream in the same recursion order (stats for the GPU driver's tests).
int ref_sampled_strategy(int D, int F, int num_iters, int max_depth, int linear_update, int seed, const float* net_w,
                         int hidden, double* strategy_out) {
  try {
    Game game(D, F);
    const int H = game.num_hands(), A = game.num_actions();
    auto params = make_params(num_iters, max_depth, linear_update, 0, 0, 0, 0);
    std::shared_ptr<IValueNet> net;
    if (net_w) net = std::make_shared<FlatNet2>(net_w, 2 + A + 2 * H, hidden, H);
    else net = create_zero_net(H, false);
    auto strategy = compute_sampled_strategy_recursive_to_leaf(game, params, net, seed);
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

// compute_stategy_stats reach weights (subgame_solving.cc:823-899): reach_probabilities[p][node][hand], dense [2][N][H].
int ref_strategy_reach(int D, int F, const double* strategy, double* reach_out) {
  try {
    Game game(D, F);
    auto tree = unroll_tree(game);
    TreeStrategy s;
    init_nd(tree.size(), game.num_hands(), game.num_actions(), 0.0, &s);
    size_t k = 0;
    for (auto& n : s) for (auto& h : n) for (double& v : h) v = strategy[k++];
    auto stats = compute_stategy_stats(game, s);
    k = 0;
    for (int p = 0; p < 2; ++p)
      for (auto& n : stats.reach_probabilities[p])
        for (double v : n) reach_out[k++] = v;
    return (int)tree.size();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// Synthetic bench/parity inputs, shared definition with rebel_b200 (SURVEY.md section 8d):
// beliefs b_p[h] = u/sum(u), u ~ U(0,1) drawn from mt19937(seed) via
// uniform_real_distribution<double>, player 0 first.
void ref_synthetic_beliefs(int H, int seed, double* out /*[2][H]*/) {
  std::mt19937 gen(seed);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  for (int p = 0; p < 2; ++p) {
    double s = 0;
    for (int h = 0; h < H; ++h) s += (out[p * H + h] = U(gen));
    for (int h = 0; h < H; ++h) out[p * H + h] /= s;
  }
}

// CPU baseline for the bench workload: `n_subgames` root subgames (seeds seed0..), each
// build_solver + multistep (subgame_solving.cc:791,666) with a TorchScript Net2 on CPU, spread
// over `threads` std::threads (one solver at a time per thread, like DataThreadLoop).
// Returns wall seconds; the caller converts to subgame-iters/s.  root_means_out optional
// [n][2][H].
double ref_bench_solve(int D, int F, int last_bid, int player_id, int num_iters, int max_depth,
                       int n_subgames, int seed0, const char* script_path, int threads,
                       double* root_means_out, const double* beliefs_in /*[n][2][H] or NULL*/) {
  try {
    torch::set_num_threads(1);
    Game game(D, F);
    const int H = game.num_hands();
    auto params = make_params(num_iters, max_depth, 1, 0, 0, 0, 0);
    std::vector<std::shared_ptr<IValueNet>> nets;
    for (int t = 0; t < threads; ++t) {
      if (script_path && script_path[0])
        nets.push_back(std::make_shared<CountingScriptNet>(script_path));
      else
        nets.push_back(create_zero_net(H, false));
    }
    std::atomic<int> next{0};
    auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t) {
      pool.emplace_back([&, t]() {
        at::set_num_threads(1);
        for (;;) {
          int i = next.fetch_add(1);
          if (i >= n_subgames) break;
          std::vector<double> b(2 * H);
          if (beliefs_in) std::copy(beliefs_in + (size_t)i * 2 * H, beliefs_in + (size_t)(i + 1) * 2 * H, b.begin());
          else ref_synthetic_beliefs(H, seed0 + i, b.data());
          auto solver = build_solver(game, PartialPublicState{last_bid, player_id},
                                     to_beliefs(b.data(), H), params, nets[t]);
          solver->multistep();
          if (root_means_out) {
            for (int p = 0; p < 2; ++p) {
              auto v = solver->get_hand_values(p);
              for (int h = 0; h < H; ++h) root_means_out[(i * 2 + p) * H + h] = v[h];
            }
          }
        }
      });
    }
    for (auto& th : pool) th.join();
    std::chrono::duration<double> dt = std::chrono::steady_clock::now() - t0;
    return dt.count();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1.0;
  }
}

// CPU baseline for self-play data generation: `threads` RlRunner loops (what
// DataThreadLoop::mainLoop does, data_loop.h:67-76) with seeds seed0+i, TorchScript Net2 on
// CPU, for `seconds` wall seconds.  Returns examples added (2 per solved subgame).
int64_t ref_bench_datagen(int D, int F, int num_iters, int max_depth, float random_action_prob,
                          int sample_leaf, const char* script_path, int threads, int seed0,
                          double seconds, double* elapsed_out) {
  try {
    torch::set_num_threads(1);
    RecursiveSolvingParams cfg;
    cfg.num_dice = D;
    cfg.num_faces = F;
    cfg.random_action_prob = random_action_prob;
    cfg.sample_leaf = sample_leaf != 0;
    cfg.subgame_params = make_params(num_iters, max_depth, 1, 0, 0, 0, 0);
    std::vector<std::shared_ptr<CountingScriptNet>> nets;
    for (int t = 0; t < threads; ++t) nets.push_back(std::make_shared<CountingScriptNet>(script_path));
    std::atomic<bool> stop{false};
    std::vector<std::thread> pool;
    auto t0 = std::chrono::steady_clock::now();
    for (int t = 0; t < threads; ++t) {
      pool.emplace_back([&, t]() {
        at::set_num_threads(1);
        RlRunner runner(cfg, nets[t], seed0 + t);
        while (!stop.load()) runner.step();
      });
    }
    // Sample the counter at the deadline (games in flight are not waited for in the rate).
    std::this_thread::sleep_for(std::chrono::duration<double>(seconds));
    int64_t n = 0;
    for (auto& net : nets) n += net->n_examples.load();
    std::chrono::duration<double> dt = std::chrono::steady_clock::now() - t0;
    if (elapsed_out) *elapsed_out = dt.count();
    stop = true;
    for (auto& th : pool) th.join();
    return n;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// The same loops timed in consecutive windows of one continuous run (the bench's --impl reference arm: one window = one
// "step"): after `warmup_s` the example counter is sampled every `window_s` seconds; counts_out[i] = examples added during
// window i.  Returns the total number of examples of the timed windows.
int64_t ref_bench_datagen_windows(int D, int F, int num_iters, int max_depth, float random_action_prob, int sample_leaf,
                                  const char* script_path, int threads, int seed0, double warmup_s, int n_windows,
                                  double window_s, int64_t* counts_out, double* seconds_out) {
  try {
    torch::set_num_threads(1);
    RecursiveSolvingParams cfg;
    cfg.num_dice = D;
    cfg.num_faces = F;
    cfg.random_action_prob = random_action_prob;
    cfg.sample_leaf = sample_leaf != 0;
    cfg.subgame_params = make_params(num_iters, max_depth, 1, 0, 0, 0, 0);
    std::vector<std::shared_ptr<CountingScriptNet>> nets;
    for (int t = 0; t < threads; ++t) nets.push_back(std::make_shared<CountingScriptNet>(script_path));
    std::atomic<bool> stop{false};
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t) {
      pool.emplace_back([&, t]() {
        at::set_num_threads(1);
        RlRunner runner(cfg, nets[t], seed0 + t);
        while (!stop.load()) runner.step();
      });
    }
    auto total = [&]() { int64_t n = 0; for (auto& net : nets) n += net->n_examples.load(); return n; };
    std::this_thread::sleep_for(std::chrono::duration<double>(warmup_s));
    int64_t prev = total(), sum = 0;
    auto t_prev = std::chrono::steady_clock::now();
    for (int i = 0; i < n_windows; ++i) {
      std::this_thread::sleep_until(t_prev + std::chrono::duration_cast<std::chrono::steady_clock::duration>(std::chrono::duration<double>(window_s)));
      const auto now = std::chrono::steady_clock::now();
      const int64_t cur = total();
      if (counts_out) counts_out[i] = cur - prev;
      if (seconds_out) seconds_out[i] = std::chrono::duration<double>(now - t_prev).count();
      sum += cur - prev;
      prev = cur;
      t_prev = now;
    }
    stop = true;
    for (auto& th : pool) th.join();
    return sum;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

}  // extern "C"
