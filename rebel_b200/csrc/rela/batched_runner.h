// BatchedRlRunner: self-play of K Liar's Dice games in lock-step on one GPU — the GPU counterpart of the reference's
// RlRunner (recursive_solving.h:40-86, recursive_solving.cc:160-275), which plays ONE game per CPU thread.
//
// A "wave" solves the current subgame of every game at once through the C ABI (include/cfrb200.h).  Two drivers:
//
//   * DEVICE walk (default): cfrb_selfplay_wave — the act_iteration draws, the sampling of the next public state, the belief
//     updates and the training examples are all produced by kernels (csrc/selfplay_kernels.cuh), every game owning a
//     std::mt19937 stream in device memory.  The loop is a software pipeline: wave w+1 is enqueued (one CUDA-graph launch)
//     BEFORE the host waits for the examples of wave w, which it hands to the sink as DEVICE pointers (the replay appends
//     them with one device-to-device copy).  The host never sees a strategy, a belief or an example.
//   * HOST walk (cfg.host_walk, parity mode): cfrb_begin_wave -> cfrb_run -> cfrb_fetch_compact, and the reference's
//     per-game code on the host with std::mt19937 itself.  Kept as the executable specification of the device walk: the tests
//     require both drivers to emit bit-identical example streams.
//
// Either way everything follows the reference's random-number draw order and fp64 belief arithmetic:
//   act_iteration ~ U{0..num_iters}                                   recursive_solving.cc:168-169
//   sample_state_to_leaf / sample_state_single                        :192-246 / :248-275
//       br_sampler ~ U{0,1}; per node eps ~ U[0,1) (float); random action or hand ~ beliefs, action ~ policy[hand]
//   belief update + eps-normalisation                                 :41-44, :235-245
//   two training examples per solved subgame                          subgame_solving.cc:672-676
// Game g of a runner seeded with s uses the generator seed s + 1 000 000 g (cfvpy/selfplay.py:250 seeds its loops with
// rank * 1000 + i, so these never collide with another loop's games), and replays the reference's RlRunner(seed = s + 10^6 g)
// exactly as long as the solver's strategies agree.
#pragma once
#include <algorithm>
#include <cstdint>
#include <functional>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../../../include/cfrb200.h"
#include "params.h"

namespace rela {

// Receives blocks of examples: q [n][Q], v [n][H] in HOST memory.  Returns false to stop the runner.
using ExampleSink = std::function<bool(const float* q, int q_dim, const float* v, int v_dim, int n)>;
// The same with DEVICE pointers on CUDA device `device` (valid until the next call of stepDevice returns).
using DeviceExampleSink = std::function<bool(const float* dev_q, int q_dim, const float* dev_v, int v_dim, int n, int device)>;

inline uint32_t game_seed(int loop_seed, int g) { return (uint32_t)loop_seed + 1000000u * (uint32_t)g; }

class BatchedRlRunner {
 public:
  BatchedRlRunner(const liars_dice::RecursiveSolvingParams& cfg, int device, int seed)
      : cfg_(cfg), K_(std::max(1, cfg.concurrent_games)), device_(device) {
    const auto& sp = cfg.subgame_params;
    cfrb_config c{};
    c.solver = sp.use_cfr ? CFRB_SOLVER_CFR : CFRB_SOLVER_FP;   // build_solver (subgame_solving.cc:791-800)
    c.optimistic = sp.optimistic;
    c.num_dice = cfg.num_dice; c.num_faces = cfg.num_faces; c.max_depth = sp.max_depth; c.num_iters = sp.num_iters;
    c.linear_update = sp.linear_update; c.dcfr = sp.dcfr; c.dcfr_alpha = sp.dcfr_alpha; c.dcfr_beta = sp.dcfr_beta;
    c.dcfr_gamma = sp.dcfr_gamma; c.max_subgames = K_; c.device = device; c.net_mode = liars_dice::effective_net_mode(cfg); c.hidden = 256;
    c.state_dtype = cfg.state_dtype;
    check(cfrb_create(&c, &h_), "cfrb_create");
    A_ = cfrb_num_actions(h_); H_ = cfrb_num_hands(h_); Q_ = cfrb_query_size(h_);
    stride_ = cfrb_table_stride(h_);
    trees_.resize(A_);   // root bids -1 .. A-2
    for (int b = -1; b <= A_ - 2; ++b) tree(b);   // built up front: the per-game walk runs on several threads and only reads them
    host_walk_ = cfg.host_walk != 0;
    ex_q_.resize((size_t)K_ * 2 * Q_); ex_v_.resize((size_t)K_ * 2 * H_);
    if (host_walk_) {
      games_.resize(K_);
      for (int g = 0; g < K_; ++g) {
        games_[g].gen.seed(game_seed(seed, g));
        resetGame(games_[g]);
      }
      last_bid_.resize(K_); player_.resize(K_); act_.resize(K_);
      beliefs_.resize((size_t)K_ * 2 * H_); snap_.resize((size_t)K_ * stride_);
    } else {
      std::vector<uint32_t> seeds(K_);
      for (int g = 0; g < K_; ++g) seeds[g] = game_seed(seed, g);
      check(cfrb_selfplay_create(h_, K_, seeds.data(), cfg.random_action_prob, cfg.sample_leaf ? 1 : 0), "cfrb_selfplay_create");
      for (int b = 0; b < 2; ++b) {   // double-buffered example hand-over
        check(cfrb_dev_alloc(device_, (size_t)K_ * 2 * Q_ * sizeof(float), (void**)&dev_q_[b]), "cfrb_dev_alloc");
        check(cfrb_dev_alloc(device_, (size_t)K_ * 2 * H_ * sizeof(float), (void**)&dev_v_[b]), "cfrb_dev_alloc");
      }
    }
  }
  ~BatchedRlRunner() {
    if (h_) {
      cfrb_sync(h_);
      for (int b = 0; b < 2; ++b) { cfrb_dev_free(device_, dev_q_[b]); cfrb_dev_free(device_, dev_v_[b]); }
      cfrb_destroy(h_);
    }
  }
  BatchedRlRunner(const BatchedRlRunner&) = delete;
  BatchedRlRunner& operator=(const BatchedRlRunner&) = delete;

  void setWeights(const std::vector<float>& flat, uint64_t version) {
    check(cfrb_set_weights(h_, flat.data(), flat.size(), version), "cfrb_set_weights");
  }
  uint64_t weightsVersion() const { return cfrb_weights_version(h_); }
  int games() const { return K_; }
  int device() const { return device_; }
  bool hostWalk() const { return host_walk_; }
  int64_t subgamesSolved() const { return subgames_solved_; }
  cfrb_handle* handle() const { return h_; }

  // One wave through the device pipeline: hands the examples of one finished wave to `sink` as device pointers while the next
  // wave is already running.  (Weights installed with setWeights take effect for the wave enqueued by the NEXT call.)
  bool stepDevice(const DeviceExampleSink& sink) {
    if (host_walk_) throw std::runtime_error("BatchedRlRunner::stepDevice needs the device walk");
    if (!started_) {       // prime the pipeline: wave 0
      check(cfrb_selfplay_wave(h_, nullptr, nullptr, 1, nullptr), "cfrb_selfplay_wave");
      started_ = true;
    }
    const int b = buf_ ^= 1;
    // finish the pending wave (examples -> dev_*_[b], games advance) and start the next one, all asynchronous
    int rows;
    if (between_waves_) {
      // ... with a stream-ordered hook in between (one process per GPU: the NCCL hand-over of the examples runs while the GPU has
      // nothing else to do, then the next wave follows on the same stream)
      rows = cfrb_selfplay_wave(h_, dev_q_[b], dev_v_[b], 0, nullptr);
      check(rows, "cfrb_selfplay_wave");
      check(cfrb_mark(h_, 6, nullptr), "cfrb_mark");
      between_waves_(dev_q_[b], dev_v_[b], rows, cfrb_handle_stream(h_));
      check(cfrb_mark(h_, 7, nullptr), "cfrb_mark");
      check(cfrb_selfplay_wave(h_, nullptr, nullptr, 1, nullptr), "cfrb_selfplay_wave");
      check(cfrb_mark_wait(h_, 7), "cfrb_mark_wait");
      float ms = 0;
      check(cfrb_mark_elapsed_ms(h_, 6, 7, &ms), "cfrb_mark_elapsed_ms");     // device time of the hook (it waits for the slowest rank)
      between_ms_sum_ += ms; between_ms_max_ = std::max(between_ms_max_, (double)ms); ++between_n_;
    } else {
      rows = cfrb_selfplay_wave(h_, dev_q_[b], dev_v_[b], 1, nullptr);
      check(rows, "cfrb_selfplay_wave");
      check(cfrb_selfplay_wait_examples(h_), "cfrb_selfplay_wait_examples");
    }
    subgames_solved_ += K_;
    return sink(dev_q_[b], Q_, dev_v_[b], H_, rows, device_);
  }
  // Hook enqueued on the handle's stream between the end of a wave (its examples are in the given device buffers) and the start
  // of the next one.
  // device time the stream spent inside the hook: (mean, max) over the waves so far, in ms
  std::pair<double, double> betweenWavesMs() const { return {between_n_ ? between_ms_sum_ / between_n_ : 0.0, between_ms_max_}; }
  void resetBetweenWavesMs() { between_ms_sum_ = between_ms_max_ = 0; between_n_ = 0; }
  void setBetweenWaves(std::function<void(const float* dev_q, const float* dev_v, int rows, void* stream)> f) { between_waves_ = std::move(f); }
  // Drain: finish the wave in flight without starting another (its examples are delivered; used at shutdown / by tests).
  bool finishDevice(const DeviceExampleSink& sink) {
    if (host_walk_ || !started_) return true;
    const int b = buf_ ^= 1;
    const int rows = cfrb_selfplay_wave(h_, dev_q_[b], dev_v_[b], 0, nullptr);
    check(rows, "cfrb_selfplay_wave");
    check(cfrb_selfplay_wait_examples(h_), "cfrb_selfplay_wait_examples");
    started_ = false;
    if (rows == 0) return true;
    subgames_solved_ += K_;
    return sink(dev_q_[b], Q_, dev_v_[b], H_, rows, device_);
  }

  // One wave delivered to `sink`, leaving the next one running (stepDevice) or, with keep_running false, no wave in flight.
  bool waveDevice(const DeviceExampleSink& sink, bool keep_running) {
    if (keep_running) return stepDevice(sink);
    if (host_walk_) throw std::runtime_error("BatchedRlRunner::waveDevice needs the device walk");
    if (!started_) {
      check(cfrb_selfplay_wave(h_, nullptr, nullptr, 1, nullptr), "cfrb_selfplay_wave");
      started_ = true;
    }
    return finishDevice(sink);
  }
  // No wave in flight: the games' states are final until the next wave, so the session can be exported or replaced.
  bool drained() const { return !started_; }
  // The session image of cfrb_selfplay_export / _import (every game's state and random stream).  A drained device walk only: the
  // host-walk parity mode keeps its games on the host and has no device session to save.
  std::string exportSession() {
    requireDrainedSession("export");
    const int64_t n = cfrb_selfplay_export(h_, nullptr, 0);
    check((int)std::min<int64_t>(n, 0), "cfrb_selfplay_export");
    std::string img((size_t)n, '\0');
    check((int)std::min<int64_t>(cfrb_selfplay_export(h_, img.data(), img.size()), 0), "cfrb_selfplay_export");
    return img;
  }
  void importSession(const std::string& img) {
    requireDrainedSession("import");
    check(cfrb_selfplay_import(h_, img.data(), img.size()), "cfrb_selfplay_import");
  }

  // One wave, examples delivered in host memory.  Device walk: a synchronous wrapper around the pipeline (tests, tools).
  bool step(const ExampleSink& sink) {
    if (!host_walk_) {
      return stepDevice([&](const float* dq, int qd, const float* dv, int vd, int n, int dev) {
        check(cfrb_dev_to_host(dev, ex_q_.data(), dq, (size_t)n * qd * sizeof(float)), "cfrb_dev_to_host");
        check(cfrb_dev_to_host(dev, ex_v_.data(), dv, (size_t)n * vd * sizeof(float)), "cfrb_dev_to_host");
        return sink(ex_q_.data(), qd, ex_v_.data(), vd, n);
      });
    }
    const int iters = cfg_.subgame_params.num_iters;
    for (int g = 0; g < K_; ++g) {
      Game& G = games_[g];
      G.act_iteration = std::uniform_int_distribution<>(0, iters)(G.gen);   // recursive_solving.cc:168-169
      last_bid_[g] = G.last_bid; player_[g] = G.player; act_[g] = G.act_iteration;
      std::copy(G.beliefs.begin(), G.beliefs.end(), beliefs_.begin() + (size_t)g * 2 * H_);
    }
    check(cfrb_begin_wave(h_, K_, last_bid_.data(), player_.data(), beliefs_.data(), act_.data()), "cfrb_begin_wave");
    check(cfrb_run(h_, iters, nullptr), "cfrb_run");
    check(cfrb_fetch_compact(h_, /*snapshot*/ 0, snap_.data()), "cfrb_fetch_compact");
    check(cfrb_examples(h_, ex_q_.data(), ex_v_.data()), "cfrb_examples");
    subgames_solved_ += K_;
    // every game owns its random stream and beliefs, so the walk is split over a few host threads without changing any result
    auto walk = [this](int g0, int g1) {
      for (int g = g0; g < g1; ++g) {
        Game& G = games_[g];
        const double* sigma = snap_.data() + (size_t)g * stride_;
        if (cfg_.sample_leaf) sampleToLeaf(G, sigma); else sampleSingle(G, sigma);
        if (G.last_bid == A_ - 1) resetGame(G);   // terminal: RlRunner::step returns, the next call starts a new game
      }
    };
    const int T = K_ >= 2048 ? 4 : 1;
    if (T == 1) {
      walk(0, K_);
    } else {
      std::vector<std::thread> th;
      for (int i = 1; i < T; ++i) th.emplace_back(walk, (int)((int64_t)K_ * i / T), (int)((int64_t)K_ * (i + 1) / T));
      walk(0, K_ / T);
      for (auto& x : th) x.join();
    }
    return sink(ex_q_.data(), Q_, ex_v_.data(), H_, 2 * K_);
  }

 private:
  struct Game {
    int last_bid = -1, player = 0, act_iteration = 0;
    std::vector<double> beliefs;   // [2][H]
    std::mt19937 gen;
  };

  void check(int rc, const char* what) {
    if (rc < 0) throw std::runtime_error(std::string(what) + ": " + cfrb_last_error());
  }
  void requireDrainedSession(const char* what) const {
    if (host_walk_)
      throw std::runtime_error(std::string("self-play session ") + what + ": the host-walk parity mode (CFRB_HOST_WALK=1) has no device "
                               "session to save or restore; use the device walk");
    if (started_) throw std::runtime_error(std::string("self-play session ") + what + ": a wave is in flight; drain the runner first");
  }
  void resetGame(Game& G) {   // recursive_solving.cc:161-163
    G.last_bid = -1; G.player = 0;
    G.beliefs.assign((size_t)2 * H_, 1.0 / H_);
  }
  const std::vector<cfrb_node>& tree(int root_bid) {
    auto& t = trees_[root_bid + 1];
    if (t.empty()) {
      t.resize(cfrb_max_nodes(h_));
      int n = cfrb_tree_template(h_, root_bid, 0, t.data(), (int)t.size());
      if (n < 0) throw std::runtime_error(cfrb_last_error());
      t.resize(n);
    }
    return t;
  }
  void bidRange(int last_bid, int* lo, int* hi) const {   // liars_dice.h:110-115
    if (last_bid < 0) { *lo = 0; *hi = A_ - 1; } else { *lo = last_bid + 1; *hi = A_; }
  }
  // normalize_beliefs_inplace (recursive_solving.cc:41-44, util.h:68-78)
  void normalize(double* b) const {
    double s = 0;
    for (int h = 0; h < H_; ++h) s += b[h] + 1e-80;
    for (int h = 0; h < H_; ++h) b[h] = (b[h] + 1e-80) / s;
  }
  // policy[hand][action] of node `n` as the reference sees it: dense over all actions, zeros outside the legal range
  double sigmaAt(const std::vector<cfrb_node>& t, const double* sigma, int n, int hand, int action) const {
    int lo, hi; bidRange(t[n].last_bid, &lo, &hi);
    if (action < lo || action >= lo + (t[n].children_end - t[n].children_begin)) return 0.0;
    const int c = t[n].children_begin + action - lo;
    return sigma[(size_t)(c - 1) * H_ + hand];
  }

  void sampleToLeaf(Game& G, const double* sigma) {   // recursive_solving.cc:192-246
    const auto& t = tree(G.last_bid);
    std::vector<std::pair<int, int>> path;
    int node = 0;
    const int br_sampler = std::uniform_int_distribution<>(0, 1)(G.gen);
    std::vector<double> sb = G.beliefs;
    std::vector<double> policy(A_);
    while (t[node].children_end - t[node].children_begin) {
      const float eps = std::uniform_real_distribution<float>(0, 1)(G.gen);
      const int pid = G.player ^ (t[node].depth & 1);
      int lo, hi; bidRange(t[node].last_bid, &lo, &hi);
      int action;
      if (pid == br_sampler && eps < cfg_.random_action_prob) {
        action = std::uniform_int_distribution<>(lo, hi - 1)(G.gen);
      } else {
        std::discrete_distribution<> hand_dis(sb.begin() + (size_t)pid * H_, sb.begin() + (size_t)(pid + 1) * H_);
        const int hand = hand_dis(G.gen);
        for (int a = 0; a < A_; ++a) policy[a] = sigmaAt(t, sigma, node, hand, a);
        std::discrete_distribution<> action_dis(policy.begin(), policy.end());
        action = action_dis(G.gen);
      }
      for (int h = 0; h < H_; ++h) sb[(size_t)pid * H_ + h] *= sigmaAt(t, sigma, node, h, action);
      normalize(sb.data() + (size_t)pid * H_);
      path.emplace_back(node, action);
      node = t[node].children_begin + action - lo;
    }
    for (auto [n, action] : path) {   // second pass with the belief-propagation strategy (== sampling strategy for CFR)
      int lo, hi; bidRange(G.last_bid, &lo, &hi);
      for (int h = 0; h < H_; ++h) G.beliefs[(size_t)G.player * H_ + h] *= sigmaAt(t, sigma, n, h, action);
      normalize(G.beliefs.data() + (size_t)G.player * H_);
      const int child = t[n].children_begin + action - lo;
      G.last_bid = t[child].last_bid;
      G.player = G.player ^ 1;
    }
  }

  void sampleSingle(Game& G, const double* sigma) {   // recursive_solving.cc:248-275
    const auto& t = tree(G.last_bid);
    const int br_sampler = std::uniform_int_distribution<>(0, 1)(G.gen);
    const float eps = std::uniform_real_distribution<float>(0, 1)(G.gen);
    int lo, hi; bidRange(G.last_bid, &lo, &hi);
    int action;
    if (G.player == br_sampler && eps < cfg_.random_action_prob) {
      action = std::uniform_int_distribution<>(lo, hi - 1)(G.gen);
    } else {
      std::discrete_distribution<> hand_dis(G.beliefs.begin() + (size_t)G.player * H_, G.beliefs.begin() + (size_t)(G.player + 1) * H_);
      const int hand = hand_dis(G.gen);
      std::vector<double> policy(A_);
      for (int a = 0; a < A_; ++a) policy[a] = sigmaAt(t, sigma, 0, hand, a);
      std::discrete_distribution<> action_dis(policy.begin(), policy.end());
      action = action_dis(G.gen);
    }
    for (int h = 0; h < H_; ++h) G.beliefs[(size_t)G.player * H_ + h] *= sigmaAt(t, sigma, 0, h, action);
    normalize(G.beliefs.data() + (size_t)G.player * H_);
    G.last_bid = action;
    G.player ^= 1;
  }

  const liars_dice::RecursiveSolvingParams cfg_;
  const int K_;
  const int device_;
  bool host_walk_ = false, started_ = false;
  double between_ms_sum_ = 0, between_ms_max_ = 0;
  int64_t between_n_ = 0;
  std::function<void(const float*, const float*, int, void*)> between_waves_;
  int buf_ = 0;
  float* dev_q_[2] = {nullptr, nullptr};
  float* dev_v_[2] = {nullptr, nullptr};
  cfrb_handle* h_ = nullptr;
  int A_ = 0, H_ = 0, Q_ = 0, stride_ = 0;
  std::vector<std::vector<cfrb_node>> trees_;
  std::vector<Game> games_;
  std::vector<int32_t> last_bid_, player_, act_;
  std::vector<double> beliefs_, snap_;
  std::vector<float> ex_q_, ex_v_;
  int64_t subgames_solved_ = 0;
};

}  // namespace rela
