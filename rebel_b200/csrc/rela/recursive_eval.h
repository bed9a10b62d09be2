// RecursiveEvaluator — BASELINE config 5: the reference's `recursive_eval --cfr --num_repeats R` (recursive_eval.cc:117-191,
// 331-363), i.e. R sampled recursive strategies (compute_sampled_strategy_recursive_to_leaf, recursive_solving.cc:301-327 with
// compute_strategy_recursive_to_leaf :76-134), their reach-weighted float32 average, and its exploitability
// (compute_exploitability2, subgame_solving.cc:802-816).
//
// The reference solves the 2^(A-2) subgames of ONE repeat depth-first on one CPU thread.  Here the subgames of MANY repeats
// are solved level by level (a subgame's root beliefs only depend on its ancestors' sampled strategies), thousands per wave
// through the C ABI.  Everything that fixes the numbers is kept: the per-repeat mt19937(seed = strategy_id) stream is consumed
// in the reference's recursion order (which depends only on the tree), a subgame solved for `act_iteration` iterations is the
// snapshot of the lock-step wave at that iteration, beliefs are propagated unnormalised inside a subgame and eps-normalised at
// its leaves, and the accumulation `sum += float(strategy) * float(reach)` runs in strategy_id order per node.
#pragma once
#include <array>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <deque>
#include <random>
#include <stdexcept>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "../../../include/cfrb200.h"
#include "params.h"

namespace rela {

// Immediate regrets read out of a handle's accumulator (cfrb_regrets_fetch): [N][H], raw sums [N][H][A] and the count.
struct ImmediateRegrets {
  std::vector<double> immediate, sums;
  int64_t count = 0;
};
inline ImmediateRegrets fetch_regrets(cfrb_handle* h, int H, int A) {
  const int N = cfrb_full_tree_nodes(h);
  if (N < 0) throw std::runtime_error(cfrb_last_error());
  ImmediateRegrets r;
  r.immediate.resize((size_t)N * H);
  r.sums.resize((size_t)N * H * A);
  if (cfrb_regrets_fetch(h, r.immediate.data(), r.sums.data(), &r.count) < 0) throw std::runtime_error(cfrb_last_error());
  return r;
}
// report_regrets' summary (recursive_eval.cc:41-52): sum of the immediate regrets of the nodes above `depth`, and of the rest.
inline std::array<double, 2> regret_summary(const std::vector<cfrb_node>& tree, const std::vector<double>& immediate, int H, int depth) {
  double top = 0, bottom = 0;
  for (size_t n = 0; n < tree.size(); ++n) {
    double s = 0;
    for (int h = 0; h < H; ++h) s += immediate[n * H + h];
    if (tree[n].depth < depth) top += s;
    else bottom += s;
  }
  return {top, bottom};
}

struct RecursiveEvalResult {
  std::vector<float> summed_strategy;   // [N][H][A]
  std::vector<float> summed_reach;      // [N][H]
  std::vector<float> final_strategy;    // summed_strategy / (summed_reach + 1e-6)   (recursive_eval.cc:362-363)
  std::vector<int> checkpoints;         // number of repeats at which exploitability was evaluated (powers of two + last)
  std::vector<std::array<double, 2>> exploitability;
  std::vector<std::array<double, 2>> ev_of_full;        // compute_ev2(full_strategy, final_strategy) per checkpoint (:368)
  std::vector<std::array<double, 2>> regret_summary;    // report_regrets' (depth < mdp_depth, rest) per checkpoint (:374-377)
  ImmediateRegrets regrets;                             // of the sampled strategies of all repeats (CFR, track_regrets)
  int num_nodes = 0;
  int64_t subgames_solved = 0;
  int64_t subgame_iters = 0;   // CFR iterations the reference would run for these subgames: the sum of their act_iterations
  double gpu_seconds = 0;   // host wall time spent inside cfrb_begin_wave / cfrb_run / cfrb_fetch_compact
};

class RecursiveEvaluator {
 public:
  RecursiveEvaluator(const liars_dice::RecursiveSolvingParams& cfg, int device, int wave_capacity)
      : cfg_(cfg), K_(std::max(1, wave_capacity)) {
    const auto& sp = cfg.subgame_params;
    const cfrb_config c = liars_dice::solver_config(cfg, device, K_);
    if (cfrb_create(&c, &h_) < 0) throw std::runtime_error(std::string("cfrb_create: ") + cfrb_last_error());
    A_ = cfrb_num_actions(h_); H_ = cfrb_num_hands(h_); stride_ = cfrb_table_stride(h_);
    // full tree + the order in which the reference's recursion creates subgame solvers (= order of its RNG draws)
    full_.resize(1 << 20);
    int n = cfrb_unroll_tree(cfg.num_dice, cfg.num_faces, -1, 0, 1 << 30, full_.data(), (int)full_.size());
    if (n < 0 || n > (int)full_.size()) throw std::runtime_error("full tree too large");
    full_.resize(n);
    visit(0);
    level_of_.assign(n, -1);
    int max_level = 0;
    for (int r : order_) { level_of_[r] = full_[r].depth / sp.max_depth; max_level = std::max(max_level, level_of_[r]); }
    by_level_.resize(max_level + 1);
    for (int r : order_) by_level_[level_of_[r]].push_back(r);
    trees_.resize(A_);
  }
  ~RecursiveEvaluator() { if (h_) cfrb_destroy(h_); }
  RecursiveEvaluator(const RecursiveEvaluator&) = delete;
  RecursiveEvaluator& operator=(const RecursiveEvaluator&) = delete;

  int numActions() const { return A_; }
  int numHands() const { return H_; }
  void setWeights(const std::vector<float>& flat) {
    if (cfrb_set_weights(h_, flat.data(), flat.size(), 1) < 0) throw std::runtime_error(cfrb_last_error());
  }

  int numNodes() const { return (int)full_.size(); }
  const std::vector<cfrb_node>& fullTree() const { return full_; }
  cfrb_handle* handle() const { return h_; }

  // compute_strategy_recursive_to_leaf with use_samplig_strategy = false (recursive_solving.cc:76-134,276-287): every subgame
  // runs all num_iters iterations; its average strategy (get_strategy) fills the inner nodes and propagates the beliefs.
  // Dense [N][H][A] fp64.
  std::vector<double> strategyToLeaf() {
    std::vector<double> out((size_t)full_.size() * H_ * A_, 0.0);
    RecursiveEvalResult scratch;
    scratch.summed_reach.assign((size_t)full_.size() * H_, 0.f);
    strategy_out_ = out.data();
    try {
      runBatch(0, 1, scratch);
    } catch (...) {
      strategy_out_ = nullptr;
      throw;
    }
    strategy_out_ = nullptr;
    return out;
  }

  // compute_strategy_recursive (recursive_solving.cc:46-74,289-299): a subgame is solved at EVERY non-terminal node of the
  // full tree; only its root row is kept, and the acting player's beliefs are updated with that row and eps-normalised.
  std::vector<double> strategyRecursive() {
    const int N = (int)full_.size(), W = 2 * H_;
    std::vector<double> out((size_t)N * H_ * A_, 0.0);
    std::vector<double> bel((size_t)N * W, 0.0);
    for (int i = 0; i < W; ++i) bel[i] = 1.0 / H_;
    for (int a = 0; a < A_; ++a) tmpl(a - 1);
    std::vector<int> level{0}, nextl;
    std::vector<int32_t> lb, pl;
    std::vector<double> b, avg;
    const int iters = cfg_.subgame_params.num_iters;
    while (!level.empty()) {
      nextl.clear();
      for (size_t off = 0; off < level.size(); off += K_) {
        const int n = (int)std::min<size_t>(K_, level.size() - off);
        lb.resize(n); pl.resize(n); b.resize((size_t)n * W); avg.resize((size_t)n * stride_);
        for (int i = 0; i < n; ++i) {
          const int node = level[off + i];
          lb[i] = full_[node].last_bid; pl[i] = full_[node].player_id;
          std::copy(bel.begin() + (size_t)node * W, bel.begin() + (size_t)(node + 1) * W, b.begin() + (size_t)i * W);
        }
        if (cfrb_begin_wave(h_, n, lb.data(), pl.data(), b.data(), nullptr) < 0) throw std::runtime_error(cfrb_last_error());
        if (cfrb_run(h_, iters, nullptr) < 0) throw std::runtime_error(cfrb_last_error());
        if (cfrb_fetch_compact(h_, 4, avg.data()) < 0) throw std::runtime_error(cfrb_last_error());
        for (int i = 0; i < n; ++i) {
          const int node = level[off + i], pid = full_[node].player_id;
          const int nc = full_[node].children_end - full_[node].children_begin;
          const int lo = full_[node].last_bid < 0 ? 0 : full_[node].last_bid + 1;
          const double* sg = avg.data() + (size_t)i * stride_;     // root row: edges 0 .. nc-1
          for (int j = 0; j < nc; ++j) {
            const int c = full_[node].children_begin + j;
            double* cb = &bel[(size_t)c * W];
            std::copy(bel.begin() + (size_t)node * W, bel.begin() + (size_t)(node + 1) * W, cb);
            for (int h = 0; h < H_; ++h) {
              const double s = sg[(size_t)j * H_ + h];
              out[((size_t)node * H_ + h) * A_ + lo + j] = s;
              cb[(size_t)pid * H_ + h] *= s;
            }
            normalize(cb + (size_t)pid * H_);
            if (full_[c].children_end != full_[c].children_begin) nextl.push_back(c);
          }
        }
      }
      level.swap(nextl);
    }
    return out;
  }

  // full_strategy (dense [N][H][A], may be null): EV of the final strategy against it at every checkpoint.  track_regrets (CFR
  // only, like the reference): immediate regrets of the sampled strategies, added to the handle's accumulator batch by batch in
  // repeat order.
  RecursiveEvalResult run(int num_repeats, int seed0, int batch_repeats, const std::vector<double>* full_strategy = nullptr,
                          bool track_regrets = false) {
    const int N = (int)full_.size();
    RecursiveEvalResult res;
    res.num_nodes = N;
    res.summed_strategy.assign((size_t)N * H_ * A_, 0.f);
    res.summed_reach.assign((size_t)N * H_, 0.f);
    if (full_strategy && full_strategy->size() != (size_t)N * H_ * A_) throw std::runtime_error("full_strategy must be [N_full][H][A]");
    track_regrets = track_regrets && cfg_.subgame_params.use_cfr;
    if (track_regrets && cfrb_regrets_reset(h_) < 0) throw std::runtime_error(cfrb_last_error());
    int done = 0;
    while (done < num_repeats) {
      // batches end at powers of two so that the exploitability curve of the reference (:364-369) can be reported
      int next_cp = 1;
      while (next_cp <= done) next_cp <<= 1;
      const int hi = std::min({num_repeats, done + std::max(1, batch_repeats), next_cp});
      if (track_regrets) sampled_.assign((size_t)(hi - done) * (N - 1) * H_, 0.f);
      runBatch(seed0 + done, hi - done, res);
      if (track_regrets) {
        if (cfrb_regrets_add(h_, sampled_.data(), hi - done) < 0) throw std::runtime_error(cfrb_last_error());
        sampled_.clear();
      }
      done = hi;
      if ((done & (done - 1)) == 0 || done == num_repeats) {
        finalize(res);
        std::vector<double> s(res.final_strategy.begin(), res.final_strategy.end());
        res.checkpoints.push_back(done);
        std::array<double, 2> e{};   // best response of both players on the GPU (cfrb_exploitability = compute_exploitability2)
        if (cfrb_exploitability(h_, s.data(), e.data()) < 0) throw std::runtime_error(cfrb_last_error());
        res.exploitability.push_back(e);
        if (full_strategy) {
          std::array<double, 2> ev{};   // compute_ev2(full_strategy, final_strategy) (:368)
          if (cfrb_ev2(h_, full_strategy->data(), s.data(), ev.data()) < 0) throw std::runtime_error(cfrb_last_error());
          res.ev_of_full.push_back(ev);
        }
        if (track_regrets) {
          res.regrets = fetch_regrets(h_, H_, A_);
          res.regret_summary.push_back(regret_summary(full_, res.regrets.immediate, H_, cfg_.subgame_params.max_depth));
        }
      }
    }
    return res;
  }

 private:
  struct Pending { int repeat, root; std::vector<double> beliefs, reach; };   // [2][H] each

  void visit(int root) {   // compute_strategy_recursive_to_leaf's control flow (recursive_solving.cc:76-134), structure only
    if (full_[root].last_bid == A_ - 1) return;
    order_.push_back(root);
    std::deque<std::pair<int, int>> q;
    q.emplace_back(root, 0);
    const int md = cfg_.subgame_params.max_depth;
    while (!q.empty()) {
      auto [fn, d] = q.front();
      q.pop_front();
      const int nc = full_[fn].children_end - full_[fn].children_begin;
      if (d < md) {
        for (int c = full_[fn].children_begin; c < full_[fn].children_end; ++c) q.emplace_back(c, d + 1);
      } else if (nc != 0) {
        visit(fn);
      }
    }
  }
  const std::vector<cfrb_node>& tmpl(int root_bid) {
    auto& t = trees_[root_bid + 1];
    if (t.empty()) {
      t.resize(cfrb_max_nodes(h_));
      int n = cfrb_tree_template(h_, root_bid, 0, t.data(), (int)t.size());
      if (n < 0) throw std::runtime_error(cfrb_last_error());
      t.resize(n);
    }
    return t;
  }
  void normalize(double* b) const {   // normalize_beliefs_inplace (recursive_solving.cc:41-44)
    double s = 0;
    for (int h = 0; h < H_; ++h) s += b[h] + 1e-80;
    for (int h = 0; h < H_; ++h) b[h] = (b[h] + 1e-80) / s;
  }

  void runBatch(int seed_first, int count, RecursiveEvalResult& res) {
    const auto& sp = cfg_.subgame_params;
    const int N = (int)full_.size();
    // act_iteration per (repeat, subgame root): discrete distribution with weight i/2+1 on even i (:304-309,315-319)
    std::vector<double> weights;
    for (int i = 0; i < sp.num_iters; ++i) weights.push_back(i % 2 ? 0.0 : (i / 2. + 1));
    std::vector<std::vector<int>> act(count, std::vector<int>(N, -1));
    const bool full_mode = strategy_out_ != nullptr;      // strategyToLeaf: no sampling, all iterations, average strategy
    for (int r = 0; r < count && !full_mode; ++r) {
      std::mt19937 gen(seed_first + r);
      for (int root : order_) {
        std::discrete_distribution<int> dist(weights.begin(), weights.end());
        act[r][root] = dist(gen);
      }
    }
    for (int a = 0; a < A_; ++a) tmpl(a - 1);     // build every template up front: the worker threads only read them
    // level 0: the game root with uniform beliefs
    std::vector<Pending> cur, next;
    for (int r = 0; r < count; ++r) cur.push_back(Pending{r, 0, std::vector<double>((size_t)2 * H_, 1.0 / H_), std::vector<double>((size_t)2 * H_, 1.0 / H_)});
    std::vector<int32_t> lb, pl, ai;
    std::vector<double> bel;
    std::vector<double> snap[2];
    while (!cur.empty()) {
      next.clear();
      // Software pipeline over the chunks of this level: the GPU solves chunk i while the host walks chunk i-1.
      size_t prev_off = 0; int prev_n = 0, slot = 0;
      for (size_t off = 0; off < cur.size(); off += K_) {
        const int n = (int)std::min<size_t>(K_, cur.size() - off);
        lb.resize(n); pl.resize(n); ai.resize(n); bel.resize((size_t)n * 2 * H_);
        int max_act = 0;
        for (int i = 0; i < n; ++i) {
          const Pending& P = cur[off + i];
          lb[i] = full_[P.root].last_bid; pl[i] = full_[P.root].player_id; ai[i] = act[P.repeat][P.root];
          max_act = std::max(max_act, full_mode ? sp.num_iters : ai[i]);
          res.subgame_iters += full_mode ? sp.num_iters : ai[i];
          std::copy(P.beliefs.begin(), P.beliefs.end(), bel.begin() + (size_t)i * 2 * H_);
        }
        const auto t0 = std::chrono::steady_clock::now();
        if (cfrb_begin_wave(h_, n, lb.data(), pl.data(), bel.data(), ai.data()) < 0) throw std::runtime_error(cfrb_last_error());
        if (cfrb_run(h_, max_act, nullptr) < 0) throw std::runtime_error(cfrb_last_error());   // asynchronous
        res.gpu_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (prev_n) expandChunk(cur, prev_off, prev_n, snap[slot ^ 1].data(), res, next);
        const auto t1 = std::chrono::steady_clock::now();
        snap[slot].resize((size_t)n * stride_);
        if (cfrb_fetch_compact(h_, full_mode ? 4 : 0, snap[slot].data()) < 0) throw std::runtime_error(cfrb_last_error());
        res.gpu_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t1).count();
        res.subgames_solved += n;
        prev_off = off; prev_n = n; slot ^= 1;
      }
      if (prev_n) expandChunk(cur, prev_off, prev_n, snap[slot ^ 1].data(), res, next);
      cur.swap(next);
    }
  }

  // Walks the solved subgames cur[off, off+n).  Subgames with the same full-tree root (different repeats) update the same
  // accumulator entries and must do so in repeat order (float32 sums, recursive_eval.cc:349-355), so the work is split by
  // root: one thread handles all repeats of a root, in order; different roots touch disjoint nodes.
  void expandChunk(const std::vector<Pending>& cur, size_t off, int n, const double* snap, RecursiveEvalResult& res,
                   std::vector<Pending>& next) {
    std::vector<int> roots;                          // distinct roots in order of first appearance
    std::vector<std::vector<int>> members;
    {
      std::vector<int> slot_of(full_.size(), -1);
      for (int i = 0; i < n; ++i) {
        const int r = cur[off + i].root;
        if (slot_of[r] < 0) { slot_of[r] = (int)roots.size(); roots.push_back(r); members.emplace_back(); }
        members[slot_of[r]].push_back(i);
      }
    }
    const int G = (int)roots.size();
    std::vector<std::vector<Pending>> out(G);
    const int T = std::max(1, std::min<int>({G, (int)std::thread::hardware_concurrency(), 16}));
    std::atomic<int> nextg{0};
    auto work = [&]() {
      std::vector<double> bel, rch;
      for (;;) {
        const int g = nextg.fetch_add(1);
        if (g >= G) break;
        for (int i : members[g]) expand(cur[off + i], snap + (size_t)i * stride_, res, out[g], bel, rch);
      }
    };
    if (T == 1) {
      work();
    } else {
      std::vector<std::thread> th;
      for (int i = 0; i < T; ++i) th.emplace_back(work);
      for (auto& x : th) x.join();
    }
    for (auto& v : out)
      for (auto& P : v) next.push_back(std::move(P));
  }

  // One solved subgame (recursive_solving.cc:97-133): accumulate strategy x reach of its inner nodes, propagate beliefs /
  // reach to its pseudo-leaves and queue the next-level subgames.  Node order = the reference's BFS = template index order
  // (parents before children), so flat per-node arrays replace its queue of belief copies.
  void expand(const Pending& P, const double* sigma, RecursiveEvalResult& res, std::vector<Pending>& next, std::vector<double>& bel,
              std::vector<double>& rch) const {
    const auto& t = trees_[full_[P.root].last_bid + 1];
    const int n_part = (int)t.size(), W = 2 * H_;
    bel.resize((size_t)n_part * W); rch.resize((size_t)n_part * W);
    std::vector<int> full_id(n_part);
    full_id[0] = P.root;
    std::copy(P.beliefs.begin(), P.beliefs.end(), bel.begin());
    std::copy(P.reach.begin(), P.reach.end(), rch.begin());
    for (int pn = 0; pn < n_part; ++pn) {
      const int fn = full_id[pn];
      const int pnc = t[pn].children_end - t[pn].children_begin;
      const int fnc = full_[fn].children_end - full_[fn].children_begin;
      const int pid = full_[fn].player_id;
      double* nb = &bel[(size_t)pn * W];
      double* nr = &rch[(size_t)pn * W];
      if (pnc == 0 && fnc != 0) {   // non-terminal leaf of the subgame: root of a subgame on the next level (:127-132)
        Pending C{P.repeat, fn, std::vector<double>(nb, nb + W), std::vector<double>(nr, nr + W)};
        normalize(C.beliefs.data());
        normalize(C.beliefs.data() + H_);
        next.push_back(std::move(C));
        continue;
      }
      // weight of infoset (node, hand) = reach_probabilities[player(node)][node][hand] under the sampled strategy
      // (recursive_eval.cc:143-148; compute_stategy_stats, subgame_solving.cc:839-842), accumulated in float32
      if (!strategy_out_)
        for (int h = 0; h < H_; ++h) res.summed_reach[(size_t)fn * H_ + h] += (float)nr[(size_t)pid * H_ + h];
      if (pnc == 0) continue;   // terminal node
      const int lo = t[pn].last_bid < 0 ? 0 : t[pn].last_bid + 1;
      for (int j = 0; j < pnc; ++j) {
        const int pc = t[pn].children_begin + j, action = lo + j;
        full_id[pc] = full_[fn].children_begin + j;
        double* cb = &bel[(size_t)pc * W];
        double* cr = &rch[(size_t)pc * W];
        std::copy(nb, nb + W, cb);
        std::copy(nr, nr + W, cr);
        // the repeat's sampled strategy as the float32 tensor of recursive_eval.cc:138-139, compact [edge = child - 1][h]
        float* samp = sampled_.empty() ? nullptr : sampled_.data() + ((size_t)P.repeat * (full_.size() - 1) + full_id[pc] - 1) * H_;
        for (int h = 0; h < H_; ++h) {
          const double s = sigma[(size_t)(pc - 1) * H_ + h];
          if (samp) samp[h] = (float)s;
          if (strategy_out_) strategy_out_[((size_t)fn * H_ + h) * A_ + action] = s;
          else res.summed_strategy[((size_t)fn * H_ + h) * A_ + action] += (float)s * (float)nr[(size_t)pid * H_ + h];
          cb[(size_t)pid * H_ + h] *= s;
          cr[(size_t)pid * H_ + h] *= s;
        }
      }
    }
  }

  void finalize(RecursiveEvalResult& res) const {
    const size_t NH = res.summed_reach.size();
    res.final_strategy.resize(res.summed_strategy.size());
    for (size_t i = 0; i < NH; ++i) {
      const float den = res.summed_reach[i] + 1e-6f;
      for (int a = 0; a < A_; ++a) res.final_strategy[i * A_ + a] = res.summed_strategy[i * A_ + a] / den;
    }
  }

  const liars_dice::RecursiveSolvingParams cfg_;
  const int K_;
  double* strategy_out_ = nullptr;   // set while strategyToLeaf() runs
  mutable std::vector<float> sampled_;   // run(track_regrets): sampled strategies of the batch's repeats, [count][N - 1][H]
  cfrb_handle* h_ = nullptr;
  int A_ = 0, H_ = 0, stride_ = 0;
  std::vector<cfrb_node> full_;
  std::vector<int> order_, level_of_;
  std::vector<std::vector<int>> by_level_;
  std::vector<std::vector<cfrb_node>> trees_;
};

}  // namespace rela
