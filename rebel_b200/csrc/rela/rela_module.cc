// Python module `rela` — drop-in for the reference's cfvpy.rela (csrc/liars_dice/rela/pybind.cc:119-213): same class and
// function names, constructor signatures, attributes and ownership (shared_ptr holders, keep_alive on pushed loops,
// subgame_params returned by reference so nested setattr from selfplay.py:604-607 works).  Underneath, one generator
// loop drives thousands of concurrent games on a GPU through libcfrb200 instead of one game on a CPU thread.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include <chrono>

#include "agent.h"
#include "batched_runner.h"
#include "cfrb_owner.h"
#include "model_locker.h"
#include "params.h"
#include "recursive_eval.h"
#include "evaluation.h"
#include "match.h"
#include "replay.h"
#include "runtime.h"

namespace py = pybind11;
using namespace rela;
using liars_dice::RecursiveSolvingParams;
using liars_dice::SubgameSolvingParams;

namespace {

// One process per GPU (torchrun): NCCL communicator of libcfrb200 (cfrb_comm_*, include/cfrb200.h).  The reference has no
// multi-process mode — its generator threads share the trainer's replay and model replicas inside one process — so this is the
// GPU counterpart of those two shared objects: ModelLocker.update_model becomes a broadcast from the trainer's rank, and a
// generator loop hands every wave's examples to the trainer rank's device-resident replay with grouped send / recv.
class Comm {
 public:
  Comm(py::bytes id, int rank, int world, int device) : device_(device) {
    const std::string s = id;
    if (s.size() != 128) throw std::runtime_error("Comm: the NCCL unique id must be 128 bytes");
    cfrb_comm* c = nullptr;
    check(cfrb_comm_create(reinterpret_cast<const uint8_t*>(s.data()), rank, world, device, &c), "cfrb_comm_create");
    c_.reset(c);
  }
  int rank() const { return cfrb_comm_rank(c_.get()); }
  int world() const { return cfrb_comm_world(c_.get()); }
  int device() const { return device_; }
  cfrb_comm* get() const { return c_.get(); }
  // flat fp32 weights (host tensor): the root's content replaces everybody else's
  void broadcastWeights(torch::Tensor flat, int root) {
    if (flat.is_cuda() || flat.scalar_type() != torch::kFloat32 || !flat.is_contiguous()) throw std::runtime_error("broadcast_weights: contiguous fp32 host tensor expected");
    py::gil_scoped_release nogil;
    check(cfrb_comm_broadcast_weights(c_.get(), flat.data_ptr<float>(), (size_t)flat.numel(), root, nullptr), "cfrb_comm_broadcast_weights");
  }
  // in-place sum of a float32 CUDA tensor over the ranks, result on the root (recursive_eval's accumulators)
  void reduceSum(torch::Tensor t, int root) {
    if (!t.is_cuda() || t.scalar_type() != torch::kFloat32 || !t.is_contiguous()) throw std::runtime_error("reduce_sum: contiguous fp32 CUDA tensor expected");
    c10::cuda::getCurrentCUDAStream(t.get_device()).synchronize();
    py::gil_scoped_release nogil;
    check(cfrb_comm_reduce_sum(c_.get(), t.data_ptr<float>(), (size_t)t.numel(), root), "cfrb_comm_reduce_sum");
  }

 private:
  CommPtr c_;
  int device_ = 0;
};

py::bytes comm_unique_id() {
  uint8_t id[128];
  check(cfrb_comm_unique_id(id), "cfrb_comm_unique_id");
  return py::bytes(reinterpret_cast<const char*>(id), 128);
}

// Communicator the generator loop created afterwards uses (None = single process): every wave's examples go to rank `root`'s
// replay, and the loops of the other ranks follow the weights of rank `root`'s ModelLocker.  ONE loop per process uses it.
std::shared_ptr<Comm> g_example_comm;
int g_example_root = 0;
void set_example_comm(std::shared_ptr<Comm> c, int root) { g_example_comm = std::move(c); g_example_root = root; }

// DataThreadLoop::mainLoop of the reference plays games one after another (rela/data_loop.h:67-76); here each loop
// iteration is one wave of `concurrent_games` subgames.  Pause / terminate are observed between waves.
class DataThreadLoop : public ThreadLoop {
 public:
  DataThreadLoop(std::shared_ptr<ModelLocker> locker, std::shared_ptr<ValuePrioritizedReplay> replay,
                 const RecursiveSolvingParams& cfg, int seed)
      : locker_(std::move(locker)), replay_(std::move(replay)), cfg_(cfg), seed_(seed), comm_(g_example_comm), comm_root_(g_example_root) {
    // configuration errors surface here, on the Python thread that builds the loop, not inside the worker
    if (cfg_.num_dice < 1 || cfg_.num_faces < 1) throw std::runtime_error("create_cfr_thread: num_dice / num_faces not set");
    if (cfg_.subgame_params.max_depth < 1 || cfg_.subgame_params.num_iters < 1)
      throw std::runtime_error("create_cfr_thread: subgame_params.max_depth and num_iters must be >= 1");
    if (cfg_.concurrent_games < 1) throw std::runtime_error("create_cfr_thread: concurrent_games must be >= 1");
  }

  void terminate() override {
    ThreadLoop::terminate();
    replay_->wake();   // a producer blocked on a full buffer re-checks terminated(); the buffer stays open for everyone else
  }

  void mainLoop() final {
    const int ndev = cfrb_device_count();
    if (ndev <= 0) throw std::runtime_error("rebel_b200: no CUDA device (there is no CPU generation path)");
    BatchedRlRunner runner(cfg_, locker_->cudaOrdinal() % ndev, seed_);
    uint64_t have = 0;
    const std::function<bool()> cancelled = [this] { return terminated(); };
    auto host_sink = [&](const float* q, int qd, const float* v, int vd, int n) { return replay_->addRows(q, qd, v, vd, n, nullptr, cancelled); };
    DevFloats recv_q, recv_v;   // collective mode, trainer rank: every rank's rows of one wave
    const bool collective = comm_ && !runner.hostWalk();
    const bool trainer_rank = !collective || comm_->rank() == comm_root_;
    // collective mode, all stream-ordered on the generator's own stream between two waves (the GPU has nothing else to do there,
    // and no NCCL kernel ever competes with a wave for SMs):
    //   1. this wave's rows of every rank -> the trainer rank's replay, device to device over NVLink (grouped send / recv);
    //   2. a vote {stop, newest weights version of the trainer rank}: all loops leave after the same wave, and all of them learn
    //      in the same wave that the trainer's ModelLocker has moved on;
    //   3. one wave after such a vote, ncclBroadcast of the trainer rank's flat weights; the other ranks install them for the
    //      wave enqueued after that (the same two-wave latency update_model has on the trainer rank's own pipelined loop + 1).
    uint64_t announced = 0, bcast_version = 0;
    bool bcast_next = false, bcast_pending = false;
    const size_t nflat = locker_->weights()->size();
    std::vector<float> flat_rx;
    if (collective) {
      const int world = comm_->world(), n = 2 * runner.games(), dev = runner.device();
      if (trainer_rank) {
        recv_q = dev_alloc(dev, (size_t)world * n * cfrb_query_size(runner.handle()));
        recv_v = dev_alloc(dev, (size_t)world * n * cfrb_num_hands(runner.handle()));
      } else {
        flat_rx.resize(nflat);
      }
      runner.setBetweenWaves([&](const float* q, const float* v, int rows, void* stream) {
        if (rows <= 0) return;
        check(cfrb_comm_gather_rows(comm_->get(), q, v, rows, cfrb_query_size(runner.handle()), cfrb_num_hands(runner.handle()), recv_q.get(),
                                    recv_v.get(), comm_root_, stream),
              "cfrb_comm_gather_rows");
        const int32_t vals[2] = {terminated() ? 1 : 0, trainer_rank ? (int32_t)locker_->version() : 0};
        check(cfrb_comm_vote(comm_->get(), vals, 2, stream), "cfrb_comm_vote");
        if (bcast_next) {
          auto w = locker_->weights();     // the trainer rank sends whatever is newest now
          check(cfrb_comm_broadcast_weights(comm_->get(), trainer_rank ? const_cast<float*>(w->data()) : nullptr, nflat, comm_root_, stream),
                "cfrb_comm_broadcast_weights");
          bcast_next = false; bcast_pending = true;
        }
      });
    }
    auto dev_sink = [&](const float* q, int qd, const float* v, int vd, int n, int dev) {
      if (!collective) return replay_->addRowsDevice(q, qd, v, vd, n, dev, cancelled);
      if (!trainer_rank) return true;
      return replay_->addRowsDevice(recv_q.get(), qd, recv_v.get(), vd, comm_->world() * n, dev, cancelled);   // gathered behind the wave (see above)
    };
    while (collective || !terminated()) {
      if (paused() && !terminated()) waitUntilResume();
      if (!collective && terminated()) break;
      const uint64_t ver = locker_->version();
      if (ver != have && (trainer_rank || have == 0)) {
        // ModelLocker::updateModel happened: install the new weights before the next wave is enqueued.  (A rank that follows the
        // trainer rank only takes its own locker's initial snapshot; later versions arrive by broadcast.)
        auto w = locker_->weights();
        runner.setWeights(*w, ver);
        have = ver;
        noteWeights(*w, ver);
      }
      const bool ok = runner.hostWalk() ? runner.step(host_sink) : runner.stepDevice(dev_sink);
      ++waves_;
      if (collective) {
        if (between_reset_.exchange(false)) runner.resetBetweenWavesMs();
        const auto bw = runner.betweenWavesMs();
        between_mean_ = bw.first; between_max_ = bw.second;
        int32_t res[2] = {0, 0};
        check(cfrb_comm_vote_result(comm_->get(), res, 2), "cfrb_comm_vote_result");
        if (bcast_pending) {
          bcast_pending = false;
          if (!trainer_rank) {
            check(cfrb_comm_broadcast_fetch(comm_->get(), flat_rx.data(), nflat), "cfrb_comm_broadcast_fetch");
            runner.setWeights(flat_rx, bcast_version);
            have = bcast_version;
            noteWeights(flat_rx, bcast_version);
          }
        }
        if ((uint64_t)res[1] > announced) { announced = (uint64_t)res[1]; bcast_version = announced; bcast_next = true; }
        if (res[0]) break;          // some rank's loop was terminated: every rank leaves after this wave
      } else if (!ok) {
        break;
      }
    }
  }

  int64_t waves() const { return waves_.load(); }
  // version / plain sum of the flat weights this loop installed last (multi-rank tests check that followers got the trainer's)
  // collective mode: device time of the stream-ordered collectives between two waves (mean, max over the waves so far; it contains
  // the wait for the slowest rank).  Reading with reset=true restarts the statistics at the next wave.
  std::pair<double, double> betweenWavesMs() const { return {between_mean_.load(), between_max_.load()}; }
  void resetBetweenWavesMs() { between_reset_ = true; }
  int64_t weightsVersion() const { return w_version_.load(); }
  double weightsChecksum() const { return w_sum_.load(); }
  int concurrentGames() const { return std::max(1, cfg_.concurrent_games); }

 private:
  std::shared_ptr<ModelLocker> locker_;
  std::shared_ptr<ValuePrioritizedReplay> replay_;
  const RecursiveSolvingParams cfg_;
  const int seed_;
  std::shared_ptr<Comm> comm_;
  const int comm_root_;
  void noteWeights(const std::vector<float>& w, uint64_t ver) {
    double acc = 0;
    for (float x : w) acc += x;
    w_sum_ = acc; w_version_ = (int64_t)ver;
  }
  std::atomic<int64_t> waves_{0};
  std::atomic<int64_t> w_version_{0};
  std::atomic<double> between_mean_{0.0}, between_max_{0.0};
  std::atomic<bool> between_reset_{false};
  std::atomic<double> w_sum_{0.0};
};

// A generator the caller drives: the BatchedRlRunner of a DataThreadLoop without the thread, so that a training loop can fix which
// waves run with which weights and the order in which their examples reach the replay (train.py --deterministic).  Each run() call
// delivers one wave; keep_running leaves the next wave running behind it (the loop's pipeline), otherwise nothing is in flight
// afterwards, which set_weights, state and load_state require.
class SelfPlayGenerator {
 public:
  SelfPlayGenerator(const RecursiveSolvingParams& cfg, int device, int seed) {
    if (cfg.num_dice < 1 || cfg.num_faces < 1) throw std::runtime_error("SelfPlayGenerator: num_dice / num_faces not set");
    if (cfg.subgame_params.max_depth < 1 || cfg.subgame_params.num_iters < 1)
      throw std::runtime_error("SelfPlayGenerator: subgame_params.max_depth and num_iters must be >= 1");
    if (cfg.concurrent_games < 1) throw std::runtime_error("SelfPlayGenerator: concurrent_games must be >= 1");
    if (cfg.host_walk)
      throw std::runtime_error("SelfPlayGenerator: the host-walk parity mode (CFRB_HOST_WALK=1) has no device session to drive, save or "
                               "restore; use the device walk");
    const int ndev = cfrb_device_count();
    if (ndev <= 0) throw std::runtime_error("rebel_b200: no CUDA device (there is no CPU generation path)");
    if (device < 0 || device >= ndev) throw std::runtime_error("SelfPlayGenerator: no CUDA device " + std::to_string(device));
    py::gil_scoped_release nogil;
    runner_ = std::make_unique<BatchedRlRunner>(cfg, device, seed);
  }

  void setWeights(torch::Tensor flat, uint64_t version) {
    requireDrained("set_weights");
    auto t = flat.to(torch::kCPU, torch::kFloat32).contiguous();
    const std::vector<float> w(t.data_ptr<float>(), t.data_ptr<float>() + t.numel());
    py::gil_scoped_release nogil;
    runner_->setWeights(w, version);
  }

  // One wave's 2 x concurrent_games examples: appended to `replay` (returns the row count) or, without one, returned as host
  // tensors (query [n, Q], values [n, H]).  A replay that cannot take the rows without blocking is an error: nothing else would
  // ever make room.
  py::object run(std::shared_ptr<ValuePrioritizedReplay> replay, bool keep_running) {
    std::vector<float> q, v;
    int rows = 0, qd = 0, vd = 0;
    {
      py::gil_scoped_release nogil;
      bool full = false;
      runner_->waveDevice([&](const float* dq, int q_dim, const float* dv, int v_dim, int n, int dev) {
        rows = n; qd = q_dim; vd = v_dim;
        if (replay) {
          full = !replay->addRowsDevice(dq, q_dim, dv, v_dim, n, dev, [] { return true; });
          return true;
        }
        q.resize((size_t)n * q_dim); v.resize((size_t)n * v_dim);
        check(cfrb_dev_to_host(dev, q.data(), dq, q.size() * sizeof(float)), "cfrb_dev_to_host");
        check(cfrb_dev_to_host(dev, v.data(), dv, v.size() * sizeof(float)), "cfrb_dev_to_host");
        return true;
      }, keep_running);
      if (full)
        throw std::runtime_error("SelfPlayGenerator.run: the replay buffer has no room for the wave's " + std::to_string(rows) +
                                 " rows (sample from it, or raise its capacity)");
    }
    if (replay) return py::int_(rows);
    auto tq = torch::empty({rows, qd}), tv = torch::empty({rows, vd});
    std::copy(q.begin(), q.end(), tq.data_ptr<float>());
    std::copy(v.begin(), v.end(), tv.data_ptr<float>());
    return py::make_tuple(tq, tv);
  }

  py::bytes state() {
    requireDrained("state");
    std::string img;
    {
      py::gil_scoped_release nogil;
      img = runner_->exportSession();
    }
    return py::bytes(img);
  }
  void loadState(py::bytes image) {
    requireDrained("load_state");
    const std::string img = image;
    py::gil_scoped_release nogil;
    runner_->importSession(img);
  }

  bool drained() const { return runner_->drained(); }
  uint64_t weightsVersion() const { return runner_->weightsVersion(); }
  int games() const { return runner_->games(); }

 private:
  void requireDrained(const char* what) const {
    if (!runner_->drained())
      throw std::runtime_error(std::string("SelfPlayGenerator.") + what + ": a wave is in flight; finish it with run(keep_running=False) first");
  }
  std::unique_ptr<BatchedRlRunner> runner_;
};

std::shared_ptr<ThreadLoop> create_cfr_thread(std::shared_ptr<ModelLocker> locker, std::shared_ptr<ValuePrioritizedReplay> replay,
                                              const RecursiveSolvingParams& cfg, int seed) {
  return std::make_shared<DataThreadLoop>(std::move(locker), std::move(replay), cfg, seed);
}

struct PhaseTimer {   // CFRB_EVAL_TIMING=1: wall time of the phases of the evaluation entry points on stderr
  std::chrono::steady_clock::time_point t = std::chrono::steady_clock::now();
  const bool on = std::getenv("CFRB_EVAL_TIMING") != nullptr;
  void lap(const char* what) {
    const auto n = std::chrono::steady_clock::now();
    if (on) std::fprintf(stderr, "[rebel_b200] %-28s %.3f s\n", what, std::chrono::duration<double>(n - t).count());
    t = n;
  }
};

int eval_device() {
  const char* e = std::getenv("CFRB_ACTOR_DEVICE");
  return e && *e ? std::atoi(e) : 0;
}

// Refusal of the device walks' game size, before a device is touched (the library refuses it too, on a handle).
void refuse_above_walk_limit(const RecursiveSolvingParams& cfg, const char* who) {
  const int A = 2 * cfg.num_dice * cfg.num_faces + 1;
  if (A > CFRB_TO_LEAF_MAX_ACTIONS)
    throw std::runtime_error(std::string(who) + ": games with more than " + std::to_string(CFRB_TO_LEAF_MAX_ACTIONS) +
                             " actions are not supported (A = " + std::to_string(A) + ": the full tree has 2^A - 1 nodes)");
}

// compute_exploitability_no_net (pybind.cc:86-104, exported as compute_exploitability_fp): the solver build_solver returns for
// params.subgame_params at the initial state, without a value net (so the tree must be full depth), with the exploitability
// printed at powers of two.  The reference never steps the solver inside its loop and returns a shadowed zero; this version
// does what the loop is written to do and returns the sum of both players' exploitabilities after num_iters iterations.  With
// fp64 tables the solve runs on the full-game solver (cfrb_full_game_*), whose checkpoints are the one-CTA full-tree solver's bit
// for bit, so games of up to CFRB_TO_LEAF_MAX_ACTIONS actions are accepted.
float compute_exploitability_fp(RecursiveSolvingParams params) {
  // unroll_tree(game, max_depth) has a leaf that is not a liar call exactly when max_depth < A: the deepest non-terminal node, the
  // sequence of all A - 1 bids, sits at depth A - 1 (subgame_solving.cc:181-184)
  const int A = 2 * params.num_dice * params.num_faces + 1;
  if (params.subgame_params.max_depth < A) throw std::runtime_error("Found a non-final leaf node, but value_net is not provided");
  py::gil_scoped_release nogil;
  const int iters = params.subgame_params.num_iters;
  std::array<double, 2> v{};
  auto checkpoints = [&](auto step, auto exploitability) {
    int done = 0;
    for (int iter = 0; iter < iters; ++iter) {
      if (((iter + 1) & iter) != 0 && iter + 1 != iters) continue;
      step(iter + 1 - done);
      done = iter + 1;
      v = exploitability();
      std::printf("Iter=%8d exploitabilities=(%.3e, %.3e) sum=%.3e\n", iter + 1, v[0], v[1], (v[0] + v[1]) / 2.);
      std::fflush(stdout);
    }
  };
  if (params.state_dtype == CFRB_STATE_F64) {
    cfrb_config c = liars_dice::solver_config(params, eval_device(), 1);
    c.net_mode = CFRB_NET_ZERO;
    cfrb_full_game* raw = nullptr;
    check(cfrb_full_game_create(&c, &raw), "cfrb_full_game_create");
    const FullGamePtr fg(raw);
    checkpoints([&](int n) { check(cfrb_full_game_step(fg.get(), n), "cfrb_full_game_step"); },
                [&] {
                  std::array<double, 2> e{};
                  check(cfrb_full_game_exploitability(fg.get(), e.data()), "cfrb_full_game_exploitability");
                  return e;
                });
  } else {   // fp32 tables: only the one-CTA full-tree solver keeps them (full trees up to 2^20 nodes)
    FullTreeSolver solver(params, eval_device(), params.subgame_params.max_depth);
    checkpoints([&](int n) { solver.step(n); }, [&] { return solver.exploitability(solver.strategy()); });
  }
  return (float)(v[0] + v[1]);
}

// compute_exploitability (pybind.cc:45-55, exported as compute_exploitability_with_net): compute_strategy_recursive with the
// checkpoint's value net, then the exploitability of the assembled full-tree strategy.  The walk and its best responses run on the
// device (cfrb_recursive_exploitability), with the strategy and best responses of the dense host walk (strategy_recursive) bit for
// bit, so games of up to CFRB_TO_LEAF_MAX_ACTIONS actions are accepted.
float compute_exploitability_with_net(RecursiveSolvingParams params, const std::string& model_path) {
  refuse_above_walk_limit(params, "compute_exploitability_with_net");
  py::gil_scoped_release nogil;
  params.net_mode = liars_dice::env_int("CFRB_EVAL_NET_MODE", CFRB_NET_FP32);   // the reference evaluates a checkpoint with an fp32 forward
  auto model = torch::jit::load(model_path, torch::kCPU);
  const HandlePtr h = open_handle(liars_dice::solver_config(params, eval_device(), 8192));
  const std::vector<float> w = flat_weights_of(model);
  check(cfrb_set_weights(h.get(), w.data(), w.size(), 1), "cfrb_set_weights");
  std::array<double, 2> e{};
  check(cfrb_recursive_exploitability(h.get(), e.data(), nullptr, nullptr, nullptr), "cfrb_recursive_exploitability");
  return (float)((e[0] + e[1]) / 2.0);
}

// compute_stats_with_net (pybind.cc:57-84): exploitability of compute_strategy_recursive_to_leaf with the net, and eval_net's MSE
// of the net against full-depth solves, with the beliefs defined by the net strategy and by the full-tree strategy.
//
// device_walk (None: above 2^20 full-tree nodes, where the dense [N][H][A] strategies are not built) takes the same numbers and
// printed lines without a dense table, for games up to CFRB_TO_LEAF_MAX_ACTIONS actions: the to-leaf walk and its best response
// on the device (cfrb_to_leaf_exploitability), the full-tree solve on the full-game solver, the candidates' reach statistics and
// each depth's root solves on an FP forest (cfrb_fp_forest_*).  The phases run one after another, each freeing its device memory.
std::tuple<float, float, float> compute_stats_device(RecursiveSolvingParams params, const std::string& model_path) {
  params.net_mode = liars_dice::env_int("CFRB_EVAL_NET_MODE", CFRB_NET_FP32);   // the reference evaluates a checkpoint with an fp32 forward
  const int device = eval_device(), A = 2 * params.num_dice * params.num_faces + 1;
  PhaseTimer pt;
  auto model = torch::jit::load(model_path, torch::kCPU);
  model.eval();
  pt.lap("load model");
  int N = 0, H = 0;
  std::vector<double> net_strategy, full_strategy;   // compact [N - 1][H]
  float exploitability = 0;
  {
    const HandlePtr h = open_handle(liars_dice::solver_config(params, device, 8192));
    const std::vector<float> w = flat_weights_of(model);
    check(cfrb_set_weights(h.get(), w.data(), w.size(), 1), "cfrb_set_weights");
    pt.lap("create evaluator");
    std::array<double, 2> e{};
    double secs[2] = {0, 0};
    check(cfrb_to_leaf_exploitability(h.get(), e.data(), nullptr, nullptr, secs), "cfrb_to_leaf_exploitability");
    exploitability = (float)((e[0] + e[1]) / 2.0);
    N = check(cfrb_full_tree_nodes(h.get()), "cfrb_full_tree_nodes");
    H = cfrb_num_hands(h.get());
    net_strategy.resize((size_t)(N - 1) * H);
    check(cfrb_to_leaf_strategy(h.get(), net_strategy.data()), "cfrb_to_leaf_strategy");
    if (pt.on) std::fprintf(stderr, "[rebel_b200] %-28s %.3f s\n[rebel_b200] %-28s %.3f s\n", "  to-leaf walk", secs[0], "  best response", secs[1]);
    pt.lap("strategy to leaf");
  }
  {
    cfrb_config c = liars_dice::solver_config(params, device, 1);
    c.net_mode = CFRB_NET_ZERO;
    cfrb_full_game* raw = nullptr;
    check(cfrb_full_game_create(&c, &raw), "cfrb_full_game_create");
    const FullGamePtr fg(raw);
    pt.lap("create full-game solver");
    check(cfrb_full_game_step(fg.get(), params.subgame_params.num_iters), "cfrb_full_game_step");
    full_strategy.resize((size_t)(N - 1) * H);
    check(cfrb_full_game_strategy(fg.get(), full_strategy.data()), "cfrb_full_game_strategy");
    pt.lap("full-game solve");
  }
  std::vector<cfrb_node> tree(N);
  if (cfrb_unroll_tree(params.num_dice, params.num_faces, -1, 0, 1 << 30, tree.data(), N) != N) throw std::runtime_error(cfrb_last_error());
  cfrb_fp_forest* raw = nullptr;
  check(cfrb_fp_forest_create(params.num_dice, params.num_faces, device, &raw), "cfrb_fp_forest_create");
  const FpForestPtr forest(raw);
  pt.lap("create forest");
  const EvalNetCandidates cand = forest_candidates(forest.get(), tree, A, H, params.subgame_params.max_depth, net_strategy, full_strategy);
  pt.lap("reach statistics");
  auto after = [&](int depth, size_t roots) {
    pt.lap(("  forest depth " + std::to_string(depth) + ", " + std::to_string(roots) + " roots").c_str());
  };
  const RootSolve solve = forest_root_solve(forest.get(), tree, H, params.subgame_params.num_iters, after);
  float mse[2];
  for (int k = 0; k < 2; ++k) {
    mse[k] = eval_net_scored(params, tree, cand, model, /*traverse_by_net=*/k == 0, /*verbose=*/true, solve);
    pt.lap(k == 0 ? "eval_net rest (net beliefs)" : "eval_net rest (full beliefs)");
  }
  return std::make_tuple(exploitability, mse[0], mse[1]);
}

std::tuple<float, float, float> compute_stats_with_net(RecursiveSolvingParams params, const std::string& model_path, py::object device_walk) {
  const int A = 2 * params.num_dice * params.num_faces + 1;
  const bool on_device = device_walk.is_none() ? ((int64_t)1 << A) - 1 > ((int64_t)1 << 20) : device_walk.cast<bool>();
  if (on_device && A > CFRB_TO_LEAF_MAX_ACTIONS)   // the library's own refusal, before a device is touched
    throw std::runtime_error("compute_stats_with_net: games with more than " + std::to_string(CFRB_TO_LEAF_MAX_ACTIONS) +
                             " actions are not supported (A = " + std::to_string(A) + ": the full tree has 2^A - 1 nodes)");
  py::gil_scoped_release nogil;
  if (on_device) return compute_stats_device(params, model_path);
  params.net_mode = liars_dice::env_int("CFRB_EVAL_NET_MODE", CFRB_NET_FP32);   // the reference evaluates a checkpoint with an fp32 forward
  PhaseTimer pt;
  auto model = torch::jit::load(model_path, torch::kCPU);
  model.eval();
  pt.lap("load model");
  std::vector<double> net_strategy;
  std::vector<cfrb_node> tree;
  float exploitability = 0;
  {
    RecursiveEvaluator ev(params, eval_device(), 8192);
    ev.setWeights(flat_weights_of(model));
    pt.lap("create evaluator");
    net_strategy = ev.strategyToLeaf();
    pt.lap("strategy to leaf");
    tree = ev.fullTree();
    std::array<double, 2> e{};
    check(cfrb_exploitability(ev.handle(), net_strategy.data(), e.data()), "cfrb_exploitability");
    exploitability = (float)((e[0] + e[1]) / 2.0);
    pt.lap("best response");
  }
  std::vector<double> full_strategy;
  {
    FullTreeSolver full(params, eval_device(), 100000);
    pt.lap("create full-tree solver");
    full.step(params.subgame_params.num_iters);
    full_strategy = full.strategy();
    pt.lap("full-tree solve");
  }
  const float mse_net = eval_net(params, eval_device(), tree, net_strategy, full_strategy, model, /*traverse_by_net=*/true, /*verbose=*/true);
  pt.lap("eval_net (net beliefs)");
  const float mse_full = eval_net(params, eval_device(), tree, net_strategy, full_strategy, model, /*traverse_by_net=*/false, /*verbose=*/true);
  pt.lap("eval_net (full beliefs)");
  return std::make_tuple(exploitability, mse_net, mse_full);
}

std::vector<float> flat_of(py::object w) {
  std::vector<float> v;
  if (!w.is_none()) {
    auto t = w.cast<torch::Tensor>().to(torch::kCPU, torch::kFloat32).contiguous();
    v.assign(t.data_ptr<float>(), t.data_ptr<float>() + t.numel());
  }
  return v;
}

// Synchronous helper for tests / benchmarks: run `waves` waves of a BatchedRlRunner on `device` and return all examples.
std::tuple<torch::Tensor, torch::Tensor> run_selfplay_waves(const RecursiveSolvingParams& cfg, int device, int seed, int waves,
                                                            py::object flat_weights) {
  const std::vector<float> w = flat_of(flat_weights);
  std::vector<float> qs, vs;
  int qd = 0, vd = 0;
  {
    py::gil_scoped_release nogil;
    BatchedRlRunner runner(cfg, device, seed);
    if (!w.empty()) runner.setWeights(w, 1);
    auto sink = [&](const float* q, int q_dim, const float* v, int v_dim, int n) {
      qd = q_dim; vd = v_dim;
      qs.insert(qs.end(), q, q + (size_t)n * q_dim);
      vs.insert(vs.end(), v, v + (size_t)n * v_dim);
      return true;
    };
    for (int i = 0; i < waves; ++i) runner.step(sink);
  }
  const int64_t n = qd ? (int64_t)(qs.size() / qd) : 0;
  auto q = torch::empty({n, qd}), v = torch::empty({n, vd});
  std::copy(qs.begin(), qs.end(), q.data_ptr<float>());
  std::copy(vs.begin(), vs.end(), v.data_ptr<float>());
  return std::make_tuple(q, v);
}

// BASELINE config 5 (`recursive_eval --cfr --num_repeats R`, recursive_eval.cc:331-369): R sampled recursive strategies,
// float32 reach-weighted average, exploitability of the average.  Returns a dict of tensors.
torch::Tensor pairs_tensor(const std::vector<std::array<double, 2>>& v) {
  auto t = torch::empty({(int64_t)v.size(), 2}, torch::kFloat64);
  for (size_t i = 0; i < v.size(); ++i) {
    t[i][0] = v[i][0];
    t[i][1] = v[i][1];
  }
  return t;
}
torch::Tensor f64_tensor(const std::vector<double>& v, std::vector<int64_t> shape) {
  auto t = torch::empty(shape, torch::kFloat64);
  std::copy(v.begin(), v.end(), t.data_ptr<double>());
  return t;
}
void put_regrets(py::dict& d, const ImmediateRegrets& r, int64_t N, int64_t H, int64_t A) {
  d["immediate_regrets"] = f64_tensor(r.immediate, {N, H});
  d["regret_sums"] = f64_tensor(r.sums, {N, H, A});
  d["regret_count"] = r.count;
}

py::dict recursive_eval_sampled(const RecursiveSolvingParams& cfg, int device, int num_repeats, int seed0, int batch_repeats,
                                int wave_capacity, py::object flat_weights, py::object full_strategy, bool track_regrets) {
  const std::vector<float> w = flat_of(flat_weights);
  std::vector<double> full;
  if (!full_strategy.is_none()) {
    auto t = full_strategy.cast<torch::Tensor>().to(torch::kCPU, torch::kFloat64).contiguous();
    full.assign(t.data_ptr<double>(), t.data_ptr<double>() + t.numel());
  }
  RecursiveEvalResult r;
  int A = 0, H = 0;
  {
    py::gil_scoped_release nogil;
    RecursiveEvaluator ev(cfg, device, wave_capacity);
    if (!w.empty()) ev.setWeights(w);
    r = ev.run(num_repeats, seed0, batch_repeats, full_strategy.is_none() ? nullptr : &full, track_regrets);
    A = ev.numActions(); H = ev.numHands();
  }
  const int64_t N = r.num_nodes;
  auto ss = torch::empty({N, H, A}), sr = torch::empty({N, H, 1}), fs = torch::empty({N, H, A});
  std::copy(r.summed_strategy.begin(), r.summed_strategy.end(), ss.data_ptr<float>());
  std::copy(r.summed_reach.begin(), r.summed_reach.end(), sr.data_ptr<float>());
  std::copy(r.final_strategy.begin(), r.final_strategy.end(), fs.data_ptr<float>());
  py::dict d;
  d["summed_strategy"] = ss; d["summed_reach"] = sr; d["final_strategy"] = fs;
  d["checkpoints"] = r.checkpoints; d["exploitability"] = pairs_tensor(r.exploitability);
  d["subgames_solved"] = r.subgames_solved; d["subgame_iters"] = r.subgame_iters;
  d["gpu_seconds"] = r.gpu_seconds;
  if (!full_strategy.is_none()) d["ev_of_full"] = pairs_tensor(r.ev_of_full);
  if (!r.regret_summary.empty()) {
    d["regret_summary"] = pairs_tensor(r.regret_summary);
    put_regrets(d, r.regrets, N, H, A);
  }
  return d;
}

// A handle that only serves the full-tree kernels (best response, EV, regrets) of one game.
struct FullTreeHandle {
  HandlePtr h;
  int A = 0, H = 0, N = 0;
  FullTreeHandle(int num_dice, int num_faces) : h(open_handle(liars_dice::full_tree_config(num_dice, num_faces, eval_device()))) {
    A = cfrb_num_actions(h.get()); H = cfrb_num_hands(h.get());
    N = check(cfrb_full_tree_nodes(h.get()), "cfrb_full_tree_nodes");
  }
  torch::Tensor dense(torch::Tensor s, const char* who) const {
    auto t = s.to(torch::kCPU, torch::kFloat64).contiguous();
    if (t.dim() != 3 || t.size(0) != N || t.size(1) != H || t.size(2) != A)
      throw std::runtime_error(std::string(who) + ": strategy must be [num_full_tree_nodes, H, A]");
    return t;
  }
};

// compute_ev2 of two compact full-tree strategies [N - 1, H] (solve_full_game's form) on the GPU: (ev0, ev1).
std::tuple<double, double> ev_of_compact_strategies(int num_dice, int num_faces, torch::Tensor s1, torch::Tensor s2) {
  FullTreeHandle f(num_dice, num_faces);
  auto a = s1.to(torch::kCPU, torch::kFloat64).contiguous(), b = s2.to(torch::kCPU, torch::kFloat64).contiguous();
  for (auto* t : {&a, &b})
    if (t->dim() != 2 || t->size(0) != f.N - 1 || t->size(1) != f.H)
      throw std::runtime_error("ev_of_compact_strategies: strategy must be [num_full_tree_nodes - 1, H]");
  std::array<double, 2> e{};
  check(cfrb_ev2_compact(f.h.get(), a.data_ptr<double>(), b.data_ptr<double>(), e.data()), "cfrb_ev2_compact");
  return std::make_tuple(e[0], e[1]);
}

// compute_ev2 (subgame_solving.cc:975-982) of two dense full-tree strategies on the GPU: (ev0, ev1).
std::tuple<double, double> ev_of_strategies(int num_dice, int num_faces, torch::Tensor s1, torch::Tensor s2) {
  FullTreeHandle f(num_dice, num_faces);
  auto a = f.dense(s1, "ev_of_strategies"), b = f.dense(s2, "ev_of_strategies");
  std::array<double, 2> e{};
  check(cfrb_ev2(f.h.get(), a.data_ptr<double>(), b.data_ptr<double>(), e.data()), "cfrb_ev2");
  return std::make_tuple(e[0], e[1]);
}

// compute_immediate_regrets (subgame_solving.cc:984-1050) of dense strategies [S][N][H][A] on the GPU, [N][H].  The strategies
// are read as float32, like the repeats recursive_eval passes through a float32 tensor (recursive_eval.cc:358); `batch` strategies
// are uploaded at a time (any batch size gives the same bits).
torch::Tensor immediate_regrets(int num_dice, int num_faces, torch::Tensor strategies, int batch) {
  FullTreeHandle f(num_dice, num_faces);
  auto s = strategies.to(torch::kCPU, torch::kFloat32).contiguous();
  if (s.dim() != 4 || s.size(1) != f.N || s.size(2) != f.H || s.size(3) != f.A)
    throw std::runtime_error("immediate_regrets: strategies must be [S, num_full_tree_nodes, H, A]");
  std::vector<cfrb_node> tree(f.N);
  if (cfrb_unroll_tree(num_dice, num_faces, -1, 0, 1 << 30, tree.data(), f.N) != f.N) throw std::runtime_error(cfrb_last_error());
  const int64_t S = s.size(0), E = (int64_t)(f.N - 1) * f.H;
  const float* dense = s.data_ptr<float>();
  check(cfrb_regrets_reset(f.h.get()), "cfrb_regrets_reset");
  std::vector<float> compact;
  batch = std::max(1, batch);
  for (int64_t off = 0; off < S; off += batch) {
    const int n = (int)std::min<int64_t>(batch, S - off);
    compact.assign((size_t)n * E, 0.f);
    for (int k = 0; k < n; ++k)
      for (int c = 1; c < f.N; ++c) {
        const int par = tree[c].parent;
        for (int h = 0; h < f.H; ++h)
          compact[(size_t)k * E + (size_t)(c - 1) * f.H + h] = dense[(((off + k) * f.N + par) * f.H + h) * f.A + tree[c].last_bid];
      }
    check(cfrb_regrets_add(f.h.get(), compact.data(), n), "cfrb_regrets_add");
  }
  return f64_tensor(fetch_regrets(f.h.get(), f.H, f.A).immediate, {f.N, f.H});
}

// The full-tree solve of recursive_eval (recursive_eval.cc:270-309): build_solver(game, params) with max_depth 100000, the
// exploitability of get_strategy() at powers of two (printed like compute_exploitability_fp) and the final get_strategy().  With
// track_regrets (CFR only), the sampling strategy after every step with an even iteration index goes into the immediate-regret
// accumulator on the device, without a host round trip.
py::dict solve_full_tree(RecursiveSolvingParams cfg, int device, bool track_regrets) {
  std::vector<int> cps;
  std::vector<std::array<double, 2>> expl;
  std::vector<double> strategy;
  ImmediateRegrets reg;
  int N = 0, H = 0, A = 0;
  const int iters = cfg.subgame_params.num_iters;
  track_regrets = track_regrets && cfg.subgame_params.use_cfr;
  {
    py::gil_scoped_release nogil;
    FullTreeSolver solver(cfg, device, 100000);
    cfrb_handle* h = solver.handle();
    N = solver.numNodes(); H = cfrb_num_hands(h); A = cfrb_num_actions(h);
    if (track_regrets) check(cfrb_regrets_reset(h), "cfrb_regrets_reset");
    int done = 0;
    for (int iter = 0; iter < iters; ++iter) {
      const bool cp = ((iter + 1) & iter) == 0 || iter + 1 == iters;
      if (track_regrets || cp) {   // without regrets the solver runs in one piece per checkpoint
        solver.step(iter + 1 - done);
        done = iter + 1;
      }
      if (track_regrets && iter % 2 == 0) check(cfrb_regrets_add_current(h), "cfrb_regrets_add_current");
      if (cp) {
        auto v = solver.exploitability(solver.strategy());
        std::printf("Iter=%8d exploitabilities=(%.3e, %.3e) sum=%.3e\n", iter + 1, v[0], v[1], (v[0] + v[1]) / 2.);
        std::fflush(stdout);
        cps.push_back(iter + 1);
        expl.push_back(v);
      }
    }
    strategy = solver.strategy();
    if (track_regrets) reg = fetch_regrets(h, H, A);
  }
  py::dict d;
  d["checkpoints"] = cps;
  d["exploitability"] = pairs_tensor(expl);
  d["strategy"] = f64_tensor(strategy, {N, H, A});
  if (track_regrets) put_regrets(d, reg, N, H, A);
  return d;
}

// solve_full_tree's solve on the whole GPU (cfrb_full_game_*): the same checkpoints, exploitabilities and printed lines, bit for
// bit, and the final average strategy in compact form [N - 1, H] (entry (child - 1) * H + hand), so that games of up to 23
// actions fit.  Times: the iterations and the best responses, host wall time around calls that synchronise.
// Nodes of the full tree above `depth` (the first level_begin[depth] in BFS order): the root, its A - 1 bids (the root cannot call)
// and C(A, d) strictly increasing action sequences of every length d >= 2.
int64_t full_tree_nodes_above(int A, int depth) {
  int64_t n = 0, c = 1;   // c = C(A, d)
  for (int d = 0; d < depth && d <= A; ++d) {
    n += d == 0 ? 1 : (d == 1 ? A - 1 : c);
    c = c * (A - d) / (d + 1);
  }
  return n;
}

py::dict solve_full_game(RecursiveSolvingParams cfg, int device, bool track_regrets, int regret_depth) {
  const int A = 2 * cfg.num_dice * cfg.num_faces + 1;
  if (A > CFRB_TO_LEAF_MAX_ACTIONS)   // the library's own refusal, before a device is touched
    throw std::runtime_error("solve_full_game: games with more than " + std::to_string(CFRB_TO_LEAF_MAX_ACTIONS) +
                             " actions are not supported (A = " + std::to_string(A) + ": the full tree has 2^A - 1 nodes)");
  std::vector<int> cps;
  std::vector<std::array<double, 2>> expl;
  std::vector<double> strategy;
  int N = 0;
  int64_t H = 1, total_bytes = 0, handle_bytes = 0;
  for (int i = 0; i < cfg.num_dice; ++i) H *= cfg.num_faces;
  double solve_s = 0, br_s = 0, total_s = 0;
  const int iters = cfg.subgame_params.num_iters;
  track_regrets = track_regrets && cfg.subgame_params.use_cfr;   // the reference tracks them for CFR only
  std::vector<double> immediate, sums, node_sums;
  int64_t regret_count = 0;
  std::array<double, 2> summary{};
  {
    py::gil_scoped_release nogil;
    const auto t0 = std::chrono::steady_clock::now();
    cfrb_config c = liars_dice::solver_config(cfg, device, 1);
    c.net_mode = CFRB_NET_ZERO;
    cfrb_full_game* raw = nullptr;
    check(cfrb_full_game_create(&c, &raw), "cfrb_full_game_create");
    const FullGamePtr fg(raw);
    N = check(cfrb_full_game_nodes(fg.get()), "cfrb_full_game_nodes");
    if (track_regrets) check(cfrb_full_game_track_regrets(fg.get()), "cfrb_full_game_track_regrets");
    check(cfrb_full_game_memory(fg.get(), &total_bytes, &handle_bytes), "cfrb_full_game_memory");
    int done = 0;
    for (int iter = 0; iter < iters; ++iter) {
      if (((iter + 1) & iter) != 0 && iter + 1 != iters) continue;   // checkpoints at powers of two and at the end
      const auto a = std::chrono::steady_clock::now();
      check(cfrb_full_game_step(fg.get(), iter + 1 - done), "cfrb_full_game_step");
      done = iter + 1;
      const auto b = std::chrono::steady_clock::now();
      std::array<double, 2> v{};
      check(cfrb_full_game_exploitability(fg.get(), v.data()), "cfrb_full_game_exploitability");
      const auto e = std::chrono::steady_clock::now();
      solve_s += std::chrono::duration<double>(b - a).count();
      br_s += std::chrono::duration<double>(e - b).count();
      std::printf("Iter=%8d exploitabilities=(%.3e, %.3e) sum=%.3e\n", iter + 1, v[0], v[1], (v[0] + v[1]) / 2.);
      std::fflush(stdout);
      cps.push_back(iter + 1);
      expl.push_back(v);
    }
    strategy.resize((size_t)(N - 1) * H);
    check(cfrb_full_game_strategy(fg.get(), strategy.data()), "cfrb_full_game_strategy");
    if (track_regrets) {
      immediate.resize((size_t)N * H); sums.resize((size_t)(N - 1) * H); node_sums.resize(N);
      check(cfrb_full_game_regrets(fg.get(), immediate.data(), sums.data(), node_sums.data(), &regret_count), "cfrb_full_game_regrets");
      // report_regrets' summary: the per-node sums over hands, added in node order (recursive_eval.h regret_summary)
      const int64_t above = full_tree_nodes_above(2 * cfg.num_dice * cfg.num_faces + 1, regret_depth);
      for (int64_t n = 0; n < N; ++n) summary[n < above ? 0 : 1] += node_sums[n];
    }
    total_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
  py::dict d;
  d["checkpoints"] = cps;
  d["exploitability"] = pairs_tensor(expl);
  d["strategy"] = f64_tensor(strategy, {(int64_t)N - 1, H});
  d["num_nodes"] = N;
  d["seconds"] = total_s; d["solve_seconds"] = solve_s; d["br_seconds"] = br_s;
  d["device_bytes"] = total_bytes; d["handle_bytes"] = handle_bytes;
  if (track_regrets) {
    d["immediate_regrets"] = f64_tensor(immediate, {(int64_t)N, H});
    d["regret_sums_compact"] = f64_tensor(sums, {(int64_t)N - 1, H});
    d["regret_count"] = regret_count;
    d["regret_summary"] = py::make_tuple(summary[0], summary[1]);
  }
  return d;
}

// compute_exploitability2 (subgame_solving.cc:802-816) of a dense full-tree strategy [N][H][A] on the GPU best-response kernel.
std::tuple<double, double> exploitability_of_strategy(int num_dice, int num_faces, torch::Tensor strategy) {
  FullTreeHandle f(num_dice, num_faces);
  auto s = f.dense(strategy, "exploitability_of_strategy");
  std::array<double, 2> e{};
  check(cfrb_exploitability(f.h.get(), s.data_ptr<double>(), e.data()), "cfrb_exploitability");
  return std::make_tuple(e[0], e[1]);
}

py::dict stats_dict(const std::vector<float>& payoff) {
  const MatchStats s = match_stats(payoff);
  py::dict d;
  d["mean"] = s.mean; d["stderr"] = s.stderr_; d["seat_means"] = std::vector<double>{s.seat[0], s.seat[1]};
  return d;
}

// CFRB_MATCH_* of a policy name ('average', 'sampled', 'every_node').
int match_policy(const std::string& policy, const char* who) {
  if (policy == "average") return CFRB_MATCH_AVERAGE;
  if (policy == "sampled") return CFRB_MATCH_SAMPLED;
  if (policy == "every_node") return CFRB_MATCH_EVERY_NODE;
  throw std::runtime_error(std::string(who) + ": policy must be 'sampled', 'average' or 'every_node' (got '" + policy + "')");
}

// A blueprint table argument as fp64 [N - 1][H] of cfg's game: a game above 23 actions and any other shape are refused.
std::vector<double> blueprint_of(py::object table, int num_dice, int num_faces, const char* who) {
  const int64_t bytes = cfrb_blueprint_bytes(num_dice, num_faces);
  if (bytes < 0) throw std::runtime_error(std::string(who) + ": " + cfrb_last_error());
  const int64_t A = 1 + 2 * (int64_t)num_dice * num_faces;
  int64_t H = 1;
  for (int i = 0; i < num_dice; ++i) H *= num_faces;
  auto t = py::module::import("torch").attr("as_tensor")(table).cast<torch::Tensor>().to(torch::kCPU, torch::kFloat64).contiguous();
  if (t.dim() != 2 || t.size(0) != ((int64_t)1 << A) - 2 || t.size(1) != H)
    throw std::runtime_error(std::string(who) + ": a blueprint of " + std::to_string(num_dice) + "x" + std::to_string(num_faces) +
                             "f is a [" + std::to_string(((int64_t)1 << A) - 2) + ", " + std::to_string(H) + "] table");
  return std::vector<double>(t.data_ptr<double>(), t.data_ptr<double>() + t.numel());
}

py::dict play_match_py(const RecursiveSolvingParams& cfg_a, const RecursiveSolvingParams& cfg_b, int device, int games, uint64_t seed,
                       const std::string& policy, py::object flat_weights_a, py::object flat_weights_b, int concurrent_games,
                       py::object policy_b, py::object blueprint_a, py::object blueprint_b) {
  const int pa = match_policy(policy, "play_match");
  const int pb = policy_b.is_none() ? pa : match_policy(policy_b.cast<std::string>(), "play_match");
  if (!blueprint_a.is_none() && !flat_weights_a.is_none())
    throw std::runtime_error("play_match: blueprint_a replaces agent A, which then has no net: flat_weights_a must be None");
  if (!blueprint_b.is_none() && !flat_weights_b.is_none())
    throw std::runtime_error("play_match: blueprint_b replaces agent B, which then has no net: flat_weights_b must be None");
  const std::vector<float> wa = flat_of(flat_weights_a), wb = flat_of(flat_weights_b);
  std::vector<double> ta, tb;
  if (!blueprint_a.is_none()) ta = blueprint_of(blueprint_a, cfg_a.num_dice, cfg_a.num_faces, "play_match");
  if (!blueprint_b.is_none()) tb = blueprint_of(blueprint_b, cfg_b.num_dice, cfg_b.num_faces, "play_match");
  MatchResult r;
  {
    py::gil_scoped_release nogil;
    r = play_match(cfg_a, cfg_b, device, games, seed, pa, wa, wb, concurrent_games, pb, blueprint_a.is_none() ? nullptr : &ta,
                   blueprint_b.is_none() ? nullptr : &tb);
  }
  py::dict d = stats_dict(r.payoff);
  auto p = torch::empty({(int64_t)games}, torch::kFloat32);
  std::copy(r.payoff.begin(), r.payoff.end(), p.data_ptr<float>());
  auto pl = torch::empty({(int64_t)games}, torch::kInt32);
  std::copy(r.plies.begin(), r.plies.end(), pl.data_ptr<int32_t>());
  d["payoff_a"] = p; d["plies"] = pl; d["solves"] = r.solves; d["subgame_iters"] = r.subgame_iters; d["seconds"] = r.seconds;
  d["solves_a"] = r.agent_solves[0]; d["solves_b"] = r.agent_solves[1];
  return d;
}

py::dict play_lbr_py(const RecursiveSolvingParams& cfg, int device, int games, uint64_t seed, py::object flat_weights, int concurrent_games,
                     int max_subgames, const std::string& policy, py::object blueprint) {
  const int pol = match_policy(policy, "play_lbr");
  if (pol == CFRB_MATCH_SAMPLED)
    throw std::runtime_error("play_lbr: policy must be 'average' or 'every_node' (LBR against the sampled policy bounds nothing: "
                             "it would respond to a drawn snapshot the agent's opponent cannot see)");
  if (!blueprint.is_none() && !flat_weights.is_none())
    throw std::runtime_error("play_lbr: a blueprint replaces the agent, which then has no net: flat_weights must be None");
  const std::vector<float> w = flat_of(flat_weights);
  std::vector<double> table;
  if (!blueprint.is_none()) table = blueprint_of(blueprint, cfg.num_dice, cfg.num_faces, "play_lbr");
  LbrResult r;
  {
    py::gil_scoped_release nogil;
    r = play_lbr(cfg, device, games, seed, w, concurrent_games, max_subgames, pol, blueprint.is_none() ? nullptr : &table);
  }
  std::vector<float> lbr(r.payoff.size());
  for (size_t i = 0; i < lbr.size(); ++i) lbr[i] = -r.payoff[i];
  const MatchStats s = match_stats(lbr);
  py::dict d;
  d["mean"] = s.mean; d["stderr"] = s.stderr_;
  d["seat_means"] = std::vector<double>{s.seat[1], s.seat[0]};   // LBR sits in seat 1 in even games, in seat 0 in odd ones
  auto p = torch::empty({(int64_t)games}, torch::kFloat32);
  std::copy(lbr.begin(), lbr.end(), p.data_ptr<float>());
  auto pl = torch::empty({(int64_t)games}, torch::kInt32);
  std::copy(r.plies.begin(), r.plies.end(), pl.data_ptr<int32_t>());
  d["payoff_lbr"] = p; d["plies"] = pl; d["solves"] = r.solves; d["whatif_solves"] = r.whatif_solves;
  d["deferred_slot_rounds"] = r.deferred_slot_rounds; d["max_subgames"] = r.capacity;
  d["subgame_iters"] = r.subgame_iters; d["seconds"] = r.seconds; d["policy"] = blueprint.is_none() ? policy : "blueprint";
  return d;
}

py::dict match_stats_py(torch::Tensor payoff) {
  auto t = payoff.to(torch::kCPU, torch::kFloat32).contiguous();
  return stats_dict(std::vector<float>(t.data_ptr<float>(), t.data_ptr<float>() + t.numel()));
}

// compute_strategy_recursive_to_leaf (recursive_solving.cc:76-134) of one agent: dense [N, H, A] fp64.
torch::Tensor strategy_recursive_to_leaf(const RecursiveSolvingParams& cfg, int device, py::object flat_weights) {
  const std::vector<float> w = flat_of(flat_weights);
  std::vector<double> s;
  int64_t N = 0, H = 0, A = 0;
  {
    py::gil_scoped_release nogil;
    RecursiveEvaluator ev(cfg, device, 8192);
    if (!w.empty()) ev.setWeights(w);
    s = ev.strategyToLeaf();
    N = ev.numNodes(); H = ev.numHands(); A = ev.numActions();
  }
  return f64_tensor(s, {N, H, A});
}

// compute_strategy_recursive (recursive_solving.cc:46-74) of one agent on the host walk (RecursiveEvaluator::strategyRecursive):
// dense [N, H, A] fp64, so the full tree is capped at 2^20 nodes.  The reference the device walk is checked against.
torch::Tensor strategy_recursive(const RecursiveSolvingParams& cfg, int device, py::object flat_weights) {
  const std::vector<float> w = flat_of(flat_weights);
  std::vector<double> s;
  int64_t N = 0, H = 0, A = 0;
  {
    py::gil_scoped_release nogil;
    RecursiveEvaluator ev(cfg, device, 8192);
    if (!w.empty()) ev.setWeights(w);
    s = ev.strategyRecursive();
    N = ev.numNodes(); H = ev.numHands(); A = ev.numActions();
  }
  return f64_tensor(s, {N, H, A});
}

// The exploitability of a policy walked and best-responded on the device by `walk` (cfrb_to_leaf_exploitability or
// cfrb_recursive_exploitability): no dense strategy, so games up to A = 23 (2x5f, 5x2f, 1x10f, 1x11f) are accepted.
using DeviceWalk = int (*)(cfrb_handle*, double*, int64_t*, int64_t*, double*);
// return_strategy adds the walked policy as the compact table [N - 1, H] (cfrb_to_leaf_strategy), a blueprint's input.
py::dict exploitability_walk(const RecursiveSolvingParams& cfg, int device, py::object flat_weights, int wave_capacity, const char* who,
                             DeviceWalk walk, const char* walk_name, bool return_strategy) {
  refuse_above_walk_limit(cfg, who);
  const std::vector<float> w = flat_of(flat_weights);
  std::array<double, 2> br{};
  double secs[2] = {0, 0}, total = 0;
  int64_t subgames = 0, iters = 0;
  int N = 0, H = 0;
  std::vector<double> strategy;
  {
    py::gil_scoped_release nogil;
    const auto t0 = std::chrono::steady_clock::now();
    const HandlePtr h = open_handle(liars_dice::solver_config(cfg, device, std::max(1, wave_capacity)));
    if (!w.empty()) check(cfrb_set_weights(h.get(), w.data(), w.size(), 1), "cfrb_set_weights");
    check(walk(h.get(), br.data(), &subgames, &iters, secs), walk_name);
    N = cfrb_full_tree_nodes(h.get());
    H = cfrb_num_hands(h.get());
    total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (return_strategy) {
      strategy.resize((size_t)(N - 1) * H);
      check(cfrb_to_leaf_strategy(h.get(), strategy.data()), "cfrb_to_leaf_strategy");
    }
  }
  py::dict d;
  d["exploitability"] = (br[0] + br[1]) / 2.;
  d["br"] = std::vector<double>{br[0], br[1]};
  d["num_nodes"] = N; d["subgames"] = subgames; d["subgame_iters"] = iters;
  d["seconds"] = total; d["walk_seconds"] = secs[0]; d["br_seconds"] = secs[1];
  if (return_strategy) d["strategy"] = f64_tensor(strategy, {(int64_t)N - 1, (int64_t)H});
  return d;
}

// The exploitability of compute_strategy_recursive_to_leaf's policy (cfrb_to_leaf_exploitability).
py::dict exploitability_to_leaf(const RecursiveSolvingParams& cfg, int device, py::object flat_weights, int wave_capacity,
                                bool return_strategy) {
  return exploitability_walk(cfg, device, flat_weights, wave_capacity, "exploitability_to_leaf", cfrb_to_leaf_exploitability,
                             "cfrb_to_leaf_exploitability", return_strategy);
}

// The exploitability of compute_strategy_recursive's every-node policy (cfrb_recursive_exploitability).
py::dict exploitability_recursive(const RecursiveSolvingParams& cfg, int device, py::object flat_weights, int wave_capacity,
                                  bool return_strategy) {
  return exploitability_walk(cfg, device, flat_weights, wave_capacity, "exploitability_recursive", cfrb_recursive_exploitability,
                             "cfrb_recursive_exploitability", return_strategy);
}

// recursive_eval's sampled evaluation (RecursiveEvaluator::run, recursive_eval.cc:331-369) walked on the device
// (cfrb_to_leaf_sampled): no dense [N, H, A] sums, so games up to A = 23 are accepted.  batch_repeats <= 0: as many repeats per
// batch as fill one wave with the largest level of subgames, between 1 and 64.
int default_batch_repeats(int A, int max_depth, int wave_capacity) {
  int64_t level = 1;
  for (int d = 0; d <= A - 1; d += max_depth) {
    int64_t c = 1;
    for (int i = 1; i <= d; ++i) c = c * (A - 1 - d + i) / i;
    level = std::max(level, c);
  }
  return (int)std::max<int64_t>(1, std::min<int64_t>(64, std::max(1, wave_capacity) / level));
}
py::dict recursive_eval_to_leaf(const RecursiveSolvingParams& cfg, int device, int num_repeats, int seed0, py::object flat_weights,
                                int wave_capacity, int batch_repeats, bool return_sums, py::object full_strategy, bool track_regrets) {
  const int A = 2 * cfg.num_dice * cfg.num_faces + 1;
  if (A > CFRB_TO_LEAF_MAX_ACTIONS)   // the library's own refusal, before a device is touched
    throw std::runtime_error("recursive_eval_to_leaf: games with more than " + std::to_string(CFRB_TO_LEAF_MAX_ACTIONS) +
                             " actions are not supported (A = " + std::to_string(A) + ": the full tree has 2^A - 1 nodes)");
  if (num_repeats < 1) throw std::runtime_error("recursive_eval_to_leaf: num_repeats must be >= 1");
  const int K = std::max(1, wave_capacity);
  const int B = batch_repeats > 0 ? batch_repeats : default_batch_repeats(A, cfg.subgame_params.max_depth, K);
  const std::vector<float> w = flat_of(flat_weights);
  std::vector<double> full;
  bool compact = false;   // full_strategy dense [N, H, A] or compact [N - 1, H], by shape
  const int64_t Hg = (int64_t)std::pow(cfg.num_faces, cfg.num_dice), Ng = ((int64_t)1 << A) - 1;
  if (!full_strategy.is_none()) {
    auto t = full_strategy.cast<torch::Tensor>().to(torch::kCPU, torch::kFloat64).contiguous();
    compact = t.dim() == 2 && t.size(0) == Ng - 1 && t.size(1) == Hg;
    if (!compact && !(t.dim() == 3 && t.size(0) == Ng && t.size(1) == Hg && t.size(2) == A))
      throw std::runtime_error("recursive_eval_to_leaf: full_strategy must be [N_full][H][A] or compact [N_full - 1][H]");
    full.assign(t.data_ptr<double>(), t.data_ptr<double>() + t.numel());
  }
  track_regrets = track_regrets && cfg.subgame_params.use_cfr;   // the reference tracks them for CFR only
  std::vector<int> cps(64);
  std::vector<double> br(128), ev(128), summary(128), immediate, rsums;
  int64_t rcount = 0;
  if (track_regrets) { immediate.resize((size_t)Ng * Hg); rsums.resize((size_t)(Ng - 1) * Hg); }
  std::vector<float> ss, sr;
  double secs[3] = {0, 0, 0}, total = 0;
  int64_t subgames = 0, iters = 0;
  int N = 0, H = 0, C = 0;
  {
    py::gil_scoped_release nogil;
    const auto t0 = std::chrono::steady_clock::now();
    const HandlePtr h = open_handle(liars_dice::solver_config(cfg, device, K));
    if (!w.empty()) check(cfrb_set_weights(h.get(), w.data(), w.size(), 1), "cfrb_set_weights");
    if (compact || track_regrets)
      C = check(cfrb_to_leaf_sampled_ev_regrets(h.get(), seed0, num_repeats, B, (int)cps.size(), cps.data(), br.data(),
                                                compact ? full.data() : nullptr, ev.data(), track_regrets, cfg.subgame_params.max_depth,
                                                summary.data(), track_regrets ? immediate.data() : nullptr,
                                                track_regrets ? rsums.data() : nullptr, &rcount, &subgames, &iters, secs),
                "cfrb_to_leaf_sampled_ev_regrets");
    if (!compact && track_regrets && !full.empty())
      throw std::runtime_error("recursive_eval_to_leaf: track_regrets takes a compact full_strategy [N_full - 1][H]");
    if (!compact && !track_regrets)
      C = check(cfrb_to_leaf_sampled(h.get(), seed0, num_repeats, B, (int)cps.size(), cps.data(), br.data(),
                                     full.empty() ? nullptr : full.data(), ev.data(), &subgames, &iters, secs),
                "cfrb_to_leaf_sampled");
    N = cfrb_full_tree_nodes(h.get());
    H = cfrb_num_hands(h.get());
    if (return_sums) {
      ss.resize((size_t)(N - 1) * H);
      sr.resize((size_t)N * H);
      check(cfrb_to_leaf_sampled_sums(h.get(), ss.data(), sr.data()), "cfrb_to_leaf_sampled_sums");
    }
    total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
  std::vector<std::array<double, 2>> e(C), evs(C);
  for (int c = 0; c < C; ++c) { e[c] = {br[2 * c], br[2 * c + 1]}; evs[c] = {ev[2 * c], ev[2 * c + 1]}; }
  py::dict d;
  d["checkpoints"] = std::vector<int>(cps.begin(), cps.begin() + C);
  d["exploitability"] = pairs_tensor(e);
  d["num_nodes"] = N; d["subgames"] = subgames; d["subgame_iters"] = iters; d["batch_repeats"] = B;
  d["seconds"] = total; d["draw_seconds"] = secs[0]; d["walk_seconds"] = secs[1]; d["br_seconds"] = secs[2];
  if (!full.empty()) d["ev_of_full"] = pairs_tensor(evs);
  if (track_regrets) {
    std::vector<std::array<double, 2>> rs(C);
    for (int c = 0; c < C; ++c) rs[c] = {summary[2 * c], summary[2 * c + 1]};
    d["regret_summary"] = pairs_tensor(rs);
    d["immediate_regrets"] = f64_tensor(immediate, {Ng, Hg});
    d["regret_sums_compact"] = f64_tensor(rsums, {Ng - 1, Hg});
    d["regret_count"] = rcount;
  }
  if (return_sums) {
    auto tss = torch::empty({(int64_t)N - 1, (int64_t)H}), tsr = torch::empty({(int64_t)N, (int64_t)H});
    std::copy(ss.begin(), ss.end(), tss.data_ptr<float>());
    std::copy(sr.begin(), sr.end(), tsr.data_ptr<float>());
    d["summed_strategy"] = tss; d["summed_reach"] = tsr;
  }
  return d;
}

// rela.Agent: index lists and actions from anything torch.as_tensor accepts (lists, numpy arrays, tensors).
std::vector<int32_t> i32_of(py::object o) {
  auto t = py::module::import("torch").attr("as_tensor")(o).cast<torch::Tensor>().to(torch::kCPU, torch::kInt32).contiguous().view(-1);
  return std::vector<int32_t>(t.data_ptr<int32_t>(), t.data_ptr<int32_t>() + t.numel());
}
torch::Tensor i32_tensor(const std::vector<int32_t>& v) {
  auto t = torch::empty({(int64_t)v.size()}, torch::kInt32);
  std::copy(v.begin(), v.end(), t.data_ptr<int32_t>());
  return t;
}

std::shared_ptr<Agent> make_agent(const RecursiveSolvingParams& cfg, int device, int tables, const std::string& policy, uint64_t seed,
                                  py::object flat_weights) {
  const int pol = match_policy(policy, "Agent");
  const std::vector<float> w = flat_of(flat_weights);
  py::gil_scoped_release nogil;
  return std::make_shared<Agent>(cfg, device, tables, pol, seed, w);
}

std::shared_ptr<Agent> make_blueprint_agent(int num_dice, int num_faces, py::object strategy, int device, int tables, uint64_t seed) {
  const std::vector<double> s = blueprint_of(strategy, num_dice, num_faces, "Agent.from_blueprint");
  py::gil_scoped_release nogil;
  return std::make_shared<Agent>(num_dice, num_faces, s, device, tables, seed);
}

void agent_new_games(Agent& a, py::object ids, py::object seats, py::object hands, py::object keys) {
  std::vector<uint64_t> k;
  if (!keys.is_none()) {
    auto t = py::module::import("torch").attr("as_tensor")(keys).cast<torch::Tensor>().to(torch::kCPU, torch::kInt64).contiguous().view(-1);
    k.assign(reinterpret_cast<const uint64_t*>(t.data_ptr<int64_t>()), reinterpret_cast<const uint64_t*>(t.data_ptr<int64_t>()) + t.numel());
  }
  a.newGames(i32_of(ids), i32_of(seats), i32_of(hands), k);
}

py::tuple agent_step(Agent& a, py::object ids, py::object actions) {
  const std::vector<int32_t> id = i32_of(ids);
  std::vector<int32_t> act = i32_of(actions), done;
  std::vector<double> probs;
  {
    py::gil_scoped_release nogil;
    a.step(id, act, probs, done);
  }
  const int64_t n = (int64_t)id.size();
  return py::make_tuple(i32_tensor(act), f64_tensor(probs, {n, (int64_t)a.numActions()}), i32_tensor(done).to(torch::kBool));
}

torch::Tensor agent_policy(Agent& a, py::object ids) {
  const std::vector<int32_t> id = i32_of(ids);
  std::vector<double> out;
  {
    py::gil_scoped_release nogil;
    out = a.policy(id);
  }
  return f64_tensor(out, {(int64_t)id.size(), (int64_t)a.numHands(), (int64_t)a.numActions()});
}

py::dict agent_state(Agent& a, py::object ids) {
  const std::vector<int32_t> id = i32_of(ids);
  const Agent::State s = a.state(id);
  py::dict d;
  d["last_bid"] = i32_tensor(s.last_bid); d["player"] = i32_tensor(s.player); d["ply"] = i32_tensor(s.ply);
  d["subgames"] = i32_tensor(s.subgames); d["act_iteration"] = i32_tensor(s.act_iteration);
  d["root_beliefs"] = f64_tensor(s.root_beliefs, {(int64_t)id.size(), 2, (int64_t)a.numHands()});
  return d;
}

py::dict agent_counts(Agent& a) {
  int64_t solves = 0, iters = 0;
  double ms = 0;
  a.counts(&solves, &iters, &ms);
  py::dict d;
  d["solves"] = solves; d["subgame_iters"] = iters; d["solve_ms"] = ms;
  return d;
}

}  // namespace

PYBIND11_MODULE(rela, m) {
  py::class_<ValueTransition, std::shared_ptr<ValueTransition>>(m, "ValueTransition")
      .def(py::init<>())
      .def_readwrite("query", &ValueTransition::query)
      .def_readwrite("values", &ValueTransition::values);

  py::class_<ValuePrioritizedReplay, std::shared_ptr<ValuePrioritizedReplay>>(m, "ValuePrioritizedReplay")
      .def(py::init<int, int, float, float, int, bool, bool>(), py::arg("capacity"), py::arg("seed"), py::arg("alpha"),
           py::arg("beta"), py::arg("prefetch"), py::arg("use_priority"), py::arg("compressed_values"))
      .def("size", &ValuePrioritizedReplay::size)
      .def("num_add", &ValuePrioritizedReplay::numAdd)
      .def("storage_device", &ValuePrioritizedReplay::storageDevice,
           "rebel_b200 extension: CUDA ordinal the rows live on (-1 host memory: no CUDA device, -2 nothing stored yet)")
      .def("sample", &ValuePrioritizedReplay::sample)
      .def("pop_until", &ValuePrioritizedReplay::popUntil)
      .def("load", &ValuePrioritizedReplay::load)
      .def("save", &ValuePrioritizedReplay::save)
      .def("extract", &ValuePrioritizedReplay::extract)
      .def("push", &ValuePrioritizedReplay::push, py::call_guard<py::gil_scoped_release>())
      .def("update_priority", &ValuePrioritizedReplay::updatePriority)
      .def("save_state", &ValuePrioritizedReplay::saveState, py::arg("path"), py::call_guard<py::gil_scoped_release>(),
           "rebel_b200 extension: write the whole state (live rows in order, weights, sum, num_add, sampler state, parameters) to "
           "`path`; refused while sampled priorities are waiting for update_priority")
      .def("load_state", &ValuePrioritizedReplay::loadState, py::arg("path"), py::arg("device") = 0,
           py::call_guard<py::gil_scoped_release>(),
           "rebel_b200 extension: restore save_state's file into this empty buffer of the same parameters (rows on CUDA `device` "
           "when one exists); later samples, sizes, eviction and blocking are the saved buffer's");

  py::class_<ThreadLoop, std::shared_ptr<ThreadLoop>>(m, "ThreadLoop");

  py::class_<SubgameSolvingParams>(m, "SubgameSolvingParams")
      .def(py::init<>())
      .def_readwrite("num_iters", &SubgameSolvingParams::num_iters)
      .def_readwrite("max_depth", &SubgameSolvingParams::max_depth)
      .def_readwrite("linear_update", &SubgameSolvingParams::linear_update)
      .def_readwrite("optimistic", &SubgameSolvingParams::optimistic)
      .def_readwrite("use_cfr", &SubgameSolvingParams::use_cfr)
      .def_readwrite("dcfr", &SubgameSolvingParams::dcfr)
      .def_readwrite("dcfr_alpha", &SubgameSolvingParams::dcfr_alpha)
      .def_readwrite("dcfr_beta", &SubgameSolvingParams::dcfr_beta)
      .def_readwrite("dcfr_gamma", &SubgameSolvingParams::dcfr_gamma);

  py::class_<RecursiveSolvingParams>(m, "RecursiveSolvingParams")
      .def(py::init<>())
      .def_readwrite("num_dice", &RecursiveSolvingParams::num_dice)
      .def_readwrite("num_faces", &RecursiveSolvingParams::num_faces)
      .def_readwrite("random_action_prob", &RecursiveSolvingParams::random_action_prob)
      .def_readwrite("sample_leaf", &RecursiveSolvingParams::sample_leaf)
      .def_readwrite("subgame_params", &RecursiveSolvingParams::subgame_params)
      // rebel_b200 extensions (defaults from CFRB_* environment variables, see params.h)
      .def_readwrite("concurrent_games", &RecursiveSolvingParams::concurrent_games)
      .def_readwrite("net_mode", &RecursiveSolvingParams::net_mode)
      .def_readwrite("state_dtype", &RecursiveSolvingParams::state_dtype)
      .def_readwrite("host_walk", &RecursiveSolvingParams::host_walk);

  py::class_<DataThreadLoop, ThreadLoop, std::shared_ptr<DataThreadLoop>>(m, "DataThreadLoop")
      .def(py::init<std::shared_ptr<ModelLocker>, std::shared_ptr<ValuePrioritizedReplay>, const RecursiveSolvingParams&, int>(),
           py::arg("model_locker"), py::arg("replay"), py::arg("params"), py::arg("thread_id"))
      .def_property_readonly("waves", &DataThreadLoop::waves, "rebel_b200 extension: waves of concurrent_games subgames completed")
      .def_property_readonly("between_waves_ms", &DataThreadLoop::betweenWavesMs,
                             "rebel_b200 extension (generator comm): (mean, max) device time in ms of the collectives between two waves")
      .def("reset_between_waves_ms", &DataThreadLoop::resetBetweenWavesMs, "restart the statistics of between_waves_ms after the wave in flight")
      .def_property_readonly("weights_version", &DataThreadLoop::weightsVersion, "rebel_b200 extension: version of the weights this loop installed last")
      .def_property_readonly("weights_checksum", &DataThreadLoop::weightsChecksum, "rebel_b200 extension: plain sum of those flat weights")
      .def_property_readonly("concurrent_games", &DataThreadLoop::concurrentGames);

  py::class_<SelfPlayGenerator, std::shared_ptr<SelfPlayGenerator>>(
      m, "SelfPlayGenerator",
      "rebel_b200 extension: the self-play of one generator loop (concurrent_games games on CUDA `device`, games seeded like "
      "create_cfr_thread's loop `seed`) driven by the caller, one wave per run() call")
      .def(py::init<const RecursiveSolvingParams&, int, int>(), py::arg("cfg"), py::arg("device"), py::arg("seed"))
      .def("set_weights", &SelfPlayGenerator::setWeights, py::arg("flat"), py::arg("version"),
           "install flat Net2 weights (FLAT_ORDER) for the waves started from now on; no wave may be in flight")
      .def("run", &SelfPlayGenerator::run, py::arg("replay") = nullptr, py::arg("keep_running") = false,
           "finish one wave (starting it first when none is in flight) and hand over its examples: appended to `replay` (returns the "
           "rows), else returned as (query, values) host tensors.  keep_running: the next wave is started before the examples are "
           "handed over and stays in flight")
      .def("state", &SelfPlayGenerator::state, "the session image (bytes: every game's state and random stream); needs no wave in flight")
      .def("load_state", &SelfPlayGenerator::loadState, py::arg("image"),
           "continue from an image of state() taken with the same game, concurrent_games and sampling parameters")
      .def_property_readonly("drained", &SelfPlayGenerator::drained, "no wave in flight")
      .def_property_readonly("weights_version", &SelfPlayGenerator::weightsVersion)
      .def_property_readonly("concurrent_games", &SelfPlayGenerator::games);

  py::class_<Context>(m, "Context")
      .def(py::init<>())
      .def("push_env_thread", &Context::pushThreadLoop, py::keep_alive<1, 2>())
      .def("start", &Context::start)
      .def("pause", &Context::pause)
      .def("resume", &Context::resume)
      .def("terminate", &Context::terminate, py::call_guard<py::gil_scoped_release>())
      .def("terminated", &Context::terminated)
      .def("error", &Context::error, "rebel_b200 extension: message of the last exception raised inside a generator loop");

  py::class_<Comm, std::shared_ptr<Comm>>(m, "Comm", "rebel_b200 extension: NCCL communicator of libcfrb200 (one process per GPU)")
      .def(py::init<py::bytes, int, int, int>(), py::arg("unique_id"), py::arg("rank"), py::arg("world"), py::arg("device"))
      .def_property_readonly("rank", &Comm::rank)
      .def_property_readonly("world", &Comm::world)
      .def("broadcast_weights", &Comm::broadcastWeights, py::arg("flat"), py::arg("root") = 0)
      .def("reduce_sum", &Comm::reduceSum, py::arg("tensor"), py::arg("root") = 0);
  m.def("comm_unique_id", &comm_unique_id, "rebel_b200 extension: ncclGetUniqueId (call on one rank, hand the 128 bytes to the others)");
  m.def("set_generator_comm", &set_example_comm, py::arg("comm"), py::arg("root") = 0,
        "rebel_b200 extension (one process per GPU): the generator loop created after this call delivers every wave's examples to "
        "rank `root`'s replay (grouped ncclSend / ncclRecv from the device buffers) and, on the other ranks, follows the weights of "
        "rank `root`'s ModelLocker (ncclBroadcast), all stream-ordered between two waves; None restores single-process behaviour.");
  m.def("set_example_comm", &set_example_comm, py::arg("comm"), py::arg("root") = 0, "alias of set_generator_comm");

  py::class_<ModelLocker, std::shared_ptr<ModelLocker>>(m, "ModelLocker")
      .def(py::init<std::vector<py::object>, const std::string&>())
      .def("update_model", &ModelLocker::updateModel)
      .def_property_readonly("version", &ModelLocker::version, "rebel_b200 extension: number of weight snapshots taken");

  m.def("compute_exploitability_fp", &compute_exploitability_fp, py::arg("params"));
  m.def("compute_exploitability_with_net", &compute_exploitability_with_net, py::arg("params"), py::arg("model_path"));
  m.def("compute_stats_with_net", &compute_stats_with_net, py::arg("params"), py::arg("model_path"), py::arg("device_walk") = py::none());
  m.def("create_cfr_thread", &create_cfr_thread, py::arg("model_locker"), py::arg("replay"), py::arg("cfg"), py::arg("seed"));
  m.def("run_selfplay_waves", &run_selfplay_waves, py::arg("cfg"), py::arg("device"), py::arg("seed"), py::arg("waves"),
        py::arg("flat_weights") = py::none(),
        "rebel_b200 extension: run `waves` waves of a BatchedRlRunner synchronously and return (queries, values).");
  m.def("exploitability_of_strategy", &exploitability_of_strategy, py::arg("num_dice"), py::arg("num_faces"), py::arg("strategy"),
        "rebel_b200 extension: compute_exploitability2 of a dense full-tree strategy (GPU best-response kernel).");
  m.def("recursive_eval_sampled", &recursive_eval_sampled, py::arg("cfg"), py::arg("device"), py::arg("num_repeats"), py::arg("seed") = 0,
        py::arg("batch_repeats") = 64, py::arg("wave_capacity") = 8192, py::arg("flat_weights") = py::none(),
        py::arg("full_strategy") = py::none(), py::arg("track_regrets") = false,
        "rebel_b200 extension: the reference's `recursive_eval --cfr --num_repeats R` (sampled recursive strategies, float32 "
        "reach-weighted average, exploitability at powers of two) with the subgame solves batched on the GPU.  full_strategy "
        "(dense [N, H, A]) adds ev_of_full [checkpoints, 2] (compute_ev2 against it); track_regrets (CFR only) adds "
        "immediate_regrets [N, H], regret_summary [checkpoints, 2] (depth < max_depth, rest), regret_sums [N, H, A] and "
        "regret_count.");
  m.def("ev_of_strategies", &ev_of_strategies, py::arg("num_dice"), py::arg("num_faces"), py::arg("s1"), py::arg("s2"),
        "rebel_b200 extension: compute_ev2 of two dense full-tree strategies (GPU kernel): (ev0, ev1).");
  m.def("ev_of_compact_strategies", &ev_of_compact_strategies, py::arg("num_dice"), py::arg("num_faces"), py::arg("s1"), py::arg("s2"),
        "rebel_b200 extension: compute_ev2(s1, s2) of two compact full-tree strategies [N - 1, H] on the GPU: (ev0, ev1).");
  m.def("immediate_regrets", &immediate_regrets, py::arg("num_dice"), py::arg("num_faces"), py::arg("strategies"),
        py::arg("batch") = 64,
        "rebel_b200 extension: compute_immediate_regrets of dense full-tree strategies [S, N, H, A] read as float32 (GPU "
        "kernels, `batch` strategies per upload): [N, H].");
  m.def("solve_full_tree", &solve_full_tree, py::arg("cfg"), py::arg("device") = 0, py::arg("track_regrets") = false,
        "rebel_b200 extension: recursive_eval's full-tree solve — dict with checkpoints, exploitability [C, 2], the final "
        "get_strategy() [N, H, A] and, with track_regrets (CFR), the immediate regrets of the sampling strategies of the "
        "even iterations (immediate_regrets, regret_sums, regret_count).");
  m.def("solve_full_game", &solve_full_game, py::arg("cfg"), py::arg("device") = 0, py::arg("track_regrets") = false,
        py::arg("regret_depth") = 2,
        "rebel_b200 extension: solve_full_tree's solve with the tree spread over the whole GPU, for games of up to 23 actions — "
        "dict with checkpoints, exploitability [C, 2] (the same bits), the final average strategy in compact form [N - 1, H] "
        "(entry (child - 1) * H + hand), num_nodes, seconds, solve_seconds, br_seconds, device_bytes and handle_bytes (device "
        "memory the solver took, and the part its handle took).  track_regrets (CFR only; ignored for FP) adds the immediate "
        "regrets of the sampling strategies of the even iterations, solve_full_tree's bits: immediate_regrets [N, H], "
        "regret_sums_compact [N - 1, H], regret_count and regret_summary (top, rest), the summed immediate regrets of the nodes "
        "above regret_depth and of the rest (report_regrets' summary).");
  m.def("play_match", &play_match_py, py::arg("cfg_a"), py::arg("cfg_b"), py::arg("device"), py::arg("games"), py::arg("seed") = 0,
        py::arg("policy") = "sampled", py::arg("flat_weights_a") = py::none(), py::arg("flat_weights_b") = py::none(),
        py::arg("concurrent_games") = 8192, py::arg("policy_b") = py::none(), py::arg("blueprint_a") = py::none(),
        py::arg("blueprint_b") = py::none(),
        "rebel_b200 extension: `games` head-to-head games (seat-swapped pairs) of agent A (cfg_a + net A) against agent B on the GPU, "
        "each re-solving subgames along the path played: A with `policy`, B with policy_b (None: the same).  'average' and "
        "'sampled' are the recursive to-leaf policies; 'every_node' re-solves at every decision (compute_strategy_recursive).  "
        "dict: payoff_a [games] (to A), plies [games], mean, stderr (over pairs), seat_means [2] (A in seat 0 / seat 1), solves, "
        "solves_a, solves_b (each agent's), subgame_iters, seconds.  blueprint_a / blueprint_b (a compact full-tree table "
        "[N - 1, H], e.g. FullGame.strategy() or exploitability_to_leaf(return_strategy=True)['strategy']) replaces that agent by "
        "a blueprint: it acts with the table's row at every node, never solves, and takes no net (refused with one) and no solver "
        "settings from its cfg.");
  m.def("play_lbr", &play_lbr_py, py::arg("cfg"), py::arg("device"), py::arg("games"), py::arg("seed") = 0,
        py::arg("flat_weights") = py::none(), py::arg("concurrent_games") = 8192, py::arg("max_subgames") = 0,
        py::arg("policy") = "average", py::arg("blueprint") = py::none(),
        "rebel_b200 extension: local best response against one agent (cfg + net) on the GPU: `games` games (seat-swapped pairs), "
        "concurrent_games at a time, at most max_subgames subgames solved per round (0: 2 x concurrent_games, at least A - 1).  "
        "The agent plays `policy`: 'average' (the recursive to-leaf policy) or 'every_node' (compute_strategy_recursive: a "
        "subgame solved at every decision; each LBR decision with a legal raise then costs 1 + m solves); 'sampled' is refused.  "
        "LBR's payoff is a lower bound on the agent's exploitability.  dict: payoff_lbr [games], plies [games], mean, stderr "
        "(over pairs), seat_means [2] (LBR in seat 0 / seat 1), solves, whatif_solves, deferred_slot_rounds, max_subgames, "
        "subgame_iters, seconds, policy.  blueprint (a compact full-tree table [N - 1, H]) plays LBR against that fixed "
        "strategy instead: no solves, no net (refused with one), policy 'blueprint'.");
  m.def("exploitability_to_leaf", &exploitability_to_leaf, py::arg("cfg"), py::arg("device") = 0, py::arg("flat_weights") = py::none(),
        py::arg("wave_capacity") = 16384, py::arg("return_strategy") = false,
        "rebel_b200 extension: exploitability of compute_strategy_recursive_to_leaf's policy (every subgame solved for num_iters "
        "iterations, get_strategy; the policy play_match's 'average' plays and play_lbr bounds), the subgames walked level by level "
        "in waves of wave_capacity and the best response taken on the GPU without a dense strategy (games with at most 23 actions "
        "whose need fits the free device memory).  dict: exploitability = (br0 + br1) / 2, br [2], num_nodes, subgames, "
        "subgame_iters, seconds, walk_seconds, br_seconds; return_strategy adds strategy, the walked policy as the compact "
        "table [N - 1, H] a blueprint plays (Agent.from_blueprint, play_match's blueprint_a / blueprint_b, play_lbr's blueprint).");
  m.def("exploitability_recursive", &exploitability_recursive, py::arg("cfg"), py::arg("device") = 0,
        py::arg("flat_weights") = py::none(), py::arg("wave_capacity") = 16384, py::arg("return_strategy") = false,
        "rebel_b200 extension: exploitability of compute_strategy_recursive's every-node policy (a subgame solved for num_iters "
        "iterations at every non-terminal node, acting with its root's average strategy; what compute_exploitability_with_net "
        "measures), the 2^(A-1) subgames walked depth by depth in waves of wave_capacity and the best response taken on the GPU "
        "without a dense strategy (games with at most 23 actions whose need fits the free device memory).  dict as "
        "exploitability_to_leaf's.");
  m.def("recursive_eval_to_leaf", &recursive_eval_to_leaf, py::arg("cfg"), py::arg("device") = 0, py::arg("num_repeats") = 1,
        py::arg("seed") = 0, py::arg("flat_weights") = py::none(), py::arg("wave_capacity") = 16384, py::arg("batch_repeats") = 0,
        py::arg("return_sums") = false, py::arg("full_strategy") = py::none(), py::arg("track_regrets") = false,
        "rebel_b200 extension: recursive_eval_sampled's evaluation (the float32 reach-weighted average of num_repeats sampled "
        "recursive strategies, strategy ids seed .. seed + num_repeats - 1, and its exploitability at every power of two and at "
        "num_repeats) with the subgames walked level by level on the device and the best responses taken there, without dense "
        "sums (games with at most 23 actions whose need fits the free device memory).  batch_repeats repeats are walked together "
        "(<= 0: enough to fill a wave, at most 64).  dict: checkpoints, exploitability [C, 2], num_nodes, subgames, subgame_iters, "
        "batch_repeats, seconds, draw_seconds, walk_seconds, br_seconds; return_sums adds the compact summed_strategy [N - 1, H] "
        "(row child - 1) and summed_reach [N, H]; full_strategy (dense [N, H, A], or compact [N - 1, H] by shape) adds ev_of_full "
        "[C, 2] (compute_ev2 against it); track_regrets (CFR only; with a compact or no full_strategy) adds the immediate regrets "
        "of the sampled strategies, recursive_eval_sampled's bits: regret_summary [C, 2] (depth < max_depth, rest), "
        "immediate_regrets [N, H], regret_sums_compact [N - 1, H] and regret_count.");
  m.def("match_stats", &match_stats_py, py::arg("payoff_a"),
        "rebel_b200 extension: play_match's mean, stderr (over the pairs 2i, 2i+1) and seat_means of a payoff vector.");
  py::class_<Agent, std::shared_ptr<Agent>>(
      m, "Agent",
      "rebel_b200 extension: a ReBeL agent (cfg + net) at `tables` independent tables, each a game against an external player, "
      "advanced one action per call on the GPU.  It plays its recursive to-leaf policy ('average' or 'sampled') along the path "
      "played, re-solving from its own beliefs at the game root and at every pseudo-leaf, or ('every_node') re-solves at every "
      "node and acts with the subgame root's average strategy; deals and seats belong to the caller.")
      .def(py::init(&make_agent), py::arg("cfg"), py::arg("device") = 0, py::arg("tables") = 8192, py::arg("policy") = "sampled",
           py::arg("seed") = 0, py::arg("flat_weights") = py::none())
      .def_static("from_blueprint", &make_blueprint_agent, py::arg("num_dice"), py::arg("num_faces"), py::arg("strategy"),
                  py::arg("device") = 0, py::arg("tables") = 8192, py::arg("seed") = 0,
                  "an agent that plays a fixed full-tree strategy: the compact table [N - 1, H] (entry [child - 1, hand]) of "
                  "FullGame.strategy(), exploitability_to_leaf(return_strategy=True) or exploitability_recursive(...).  It never "
                  "solves; its draws are the same (seed, key) streams as any Agent's, so the table of an 'average' agent's walked "
                  "policy answers as that agent")
      .def("new_games", &agent_new_games, py::arg("ids"), py::arg("seats"), py::arg("hands"), py::arg("keys") = py::none(),
           "start a game at each listed table: the agent in seat seats[i] (0 moves first) with hand hands[i]; keys[i] keys the "
           "game's random stream (None: the number of games started before, in list order)")
      .def("step", &agent_step, py::arg("ids"), py::arg("actions"),
           "one action at each listed table: actions[i] is applied (normally the opponent's; on the agent's turn it overrides the "
           "agent), -1 lets the agent play.  Returns (actions played int32 [n], probs float64 [n, A]: the agent's row for its hand "
           "on its turns, NaN on the opponent's, done bool [n]: the liar call ended the game)")
      .def("policy", &agent_policy, py::arg("ids"),
           "the agent's strategy for the player to move at each listed table: float64 [n, H, A], 0 on illegal actions")
      .def("state", &agent_state, py::arg("ids"),
           "dict of last_bid, player, ply, subgames, act_iteration [n] and root_beliefs [n, 2, H] of the current subgame")
      .def("counts", &agent_counts, "dict: solves, subgame_iters, solve_ms (device time of the solves) since creation")
      .def("close", &Agent::close, "release the agent and its handle")
      .def_property_readonly("num_actions", &Agent::numActions)
      .def_property_readonly("num_hands", &Agent::numHands)
      .def_property_readonly("tables", &Agent::tables);
  m.def("strategy_recursive_to_leaf", &strategy_recursive_to_leaf, py::arg("cfg"), py::arg("device") = 0,
        py::arg("flat_weights") = py::none(),
        "rebel_b200 extension: compute_strategy_recursive_to_leaf (every subgame solved for num_iters iterations, get_strategy) as a "
        "dense full-tree strategy [N, H, A] fp64 (games whose full tree has at most 2^20 nodes).");
  m.def("strategy_recursive", &strategy_recursive, py::arg("cfg"), py::arg("device") = 0, py::arg("flat_weights") = py::none(),
        "rebel_b200 extension: compute_strategy_recursive (a subgame solved for num_iters iterations at every non-terminal node, its "
        "root row kept) on the host walk, as a dense full-tree strategy [N, H, A] fp64 (games whose full tree has at most 2^20 "
        "nodes): the reference of exploitability_recursive.");
}
