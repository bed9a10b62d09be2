// Python module `rela` — drop-in for the reference's cfvpy.rela (csrc/liars_dice/rela/pybind.cc:119-213): same class and
// function names, constructor signatures, attributes and ownership (shared_ptr holders, keep_alive on pushed loops,
// subgame_params returned by reference so nested setattr from selfplay.py:604-607 works).  Underneath, one generator
// loop drives thousands of concurrent games on a GPU through libcfrb200 instead of one game on a CPU thread.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include <chrono>

#include "batched_runner.h"
#include "model_locker.h"
#include "params.h"
#include "recursive_eval.h"
#include "evaluation.h"
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
    if (cfrb_comm_create(reinterpret_cast<const uint8_t*>(s.data()), rank, world, device, &c_) < 0)
      throw std::runtime_error(std::string("cfrb_comm_create: ") + cfrb_last_error());
  }
  ~Comm() { if (c_) cfrb_comm_destroy(c_); }
  Comm(const Comm&) = delete;
  Comm& operator=(const Comm&) = delete;
  int rank() const { return cfrb_comm_rank(c_); }
  int world() const { return cfrb_comm_world(c_); }
  int device() const { return device_; }
  cfrb_comm* get() const { return c_; }
  // flat fp32 weights (host tensor): the root's content replaces everybody else's
  void broadcastWeights(torch::Tensor flat, int root) {
    if (flat.is_cuda() || flat.scalar_type() != torch::kFloat32 || !flat.is_contiguous()) throw std::runtime_error("broadcast_weights: contiguous fp32 host tensor expected");
    py::gil_scoped_release nogil;
    if (cfrb_comm_broadcast_weights(c_, flat.data_ptr<float>(), (size_t)flat.numel(), root, nullptr) < 0) throw std::runtime_error(cfrb_last_error());
  }
  // in-place sum of a float32 CUDA tensor over the ranks, result on the root (recursive_eval's accumulators)
  void reduceSum(torch::Tensor t, int root) {
    if (!t.is_cuda() || t.scalar_type() != torch::kFloat32 || !t.is_contiguous()) throw std::runtime_error("reduce_sum: contiguous fp32 CUDA tensor expected");
    c10::cuda::getCurrentCUDAStream(t.get_device()).synchronize();
    py::gil_scoped_release nogil;
    if (cfrb_comm_reduce_sum(c_, t.data_ptr<float>(), (size_t)t.numel(), root) < 0) throw std::runtime_error(cfrb_last_error());
  }

 private:
  cfrb_comm* c_ = nullptr;
  int device_ = 0;
};

py::bytes comm_unique_id() {
  uint8_t id[128];
  if (cfrb_comm_unique_id(id) < 0) throw std::runtime_error(std::string("cfrb_comm_unique_id: ") + cfrb_last_error());
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
    float* recv_q = nullptr; float* recv_v = nullptr;
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
        if (cfrb_dev_alloc(dev, (size_t)world * n * cfrb_query_size(runner.handle()) * sizeof(float), (void**)&recv_q) < 0 ||
            cfrb_dev_alloc(dev, (size_t)world * n * cfrb_num_hands(runner.handle()) * sizeof(float), (void**)&recv_v) < 0)
          throw std::runtime_error(cfrb_last_error());
      } else {
        flat_rx.resize(nflat);
      }
      runner.setBetweenWaves([&](const float* q, const float* v, int rows, void* stream) {
        if (rows <= 0) return;
        if (cfrb_comm_gather_rows(comm_->get(), q, v, rows, cfrb_query_size(runner.handle()), cfrb_num_hands(runner.handle()), recv_q, recv_v,
                                  comm_root_, stream) < 0)
          throw std::runtime_error(cfrb_last_error());
        const int32_t vals[2] = {terminated() ? 1 : 0, trainer_rank ? (int32_t)locker_->version() : 0};
        if (cfrb_comm_vote(comm_->get(), vals, 2, stream) < 0) throw std::runtime_error(cfrb_last_error());
        if (bcast_next) {
          auto w = locker_->weights();     // the trainer rank sends whatever is newest now
          if (cfrb_comm_broadcast_weights(comm_->get(), trainer_rank ? const_cast<float*>(w->data()) : nullptr, nflat, comm_root_, stream) < 0)
            throw std::runtime_error(cfrb_last_error());
          bcast_next = false; bcast_pending = true;
        }
      });
    }
    auto dev_sink = [&](const float* q, int qd, const float* v, int vd, int n, int dev) {
      if (!collective) return replay_->addRowsDevice(q, qd, v, vd, n, dev, cancelled);
      if (!trainer_rank) return true;
      return replay_->addRowsDevice(recv_q, qd, recv_v, vd, comm_->world() * n, dev, cancelled);   // gathered behind the wave (see above)
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
        if (cfrb_comm_vote_result(comm_->get(), res, 2) < 0) throw std::runtime_error(cfrb_last_error());
        if (bcast_pending) {
          bcast_pending = false;
          if (!trainer_rank) {
            if (cfrb_comm_broadcast_fetch(comm_->get(), flat_rx.data(), nflat) < 0) throw std::runtime_error(cfrb_last_error());
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
    if (recv_q) { cfrb_dev_free(runner.device(), recv_q); cfrb_dev_free(runner.device(), recv_v); }
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

// compute_exploitability_no_net (pybind.cc:86-104, exported as compute_exploitability_fp): the solver build_solver returns for
// params.subgame_params at the initial state, without a value net (so the tree must be full depth), with the exploitability
// printed at powers of two.  The reference never steps the solver inside its loop and returns a shadowed zero; this version
// does what the loop is written to do and returns the sum of both players' exploitabilities after num_iters iterations.
float compute_exploitability_fp(RecursiveSolvingParams params) {
  py::gil_scoped_release nogil;
  FullTreeSolver solver(params, eval_device(), params.subgame_params.max_depth);
  std::array<double, 2> v{};
  int done = 0;
  for (int iter = 0; iter < params.subgame_params.num_iters; ++iter) {
    if (((iter + 1) & iter) == 0 || iter + 1 == params.subgame_params.num_iters) {
      solver.step(iter + 1 - done);
      done = iter + 1;
      v = solver.exploitability(solver.strategy());
      std::printf("Iter=%8d exploitabilities=(%.3e, %.3e) sum=%.3e\n", iter + 1, v[0], v[1], (v[0] + v[1]) / 2.);
    }
  }
  return (float)(v[0] + v[1]);
}

// compute_exploitability (pybind.cc:45-55, exported as compute_exploitability_with_net): compute_strategy_recursive with the
// checkpoint's value net, then the exploitability of the assembled full-tree strategy.
float compute_exploitability_with_net(RecursiveSolvingParams params, const std::string& model_path) {
  py::gil_scoped_release nogil;
  params.net_mode = liars_dice::env_int("CFRB_EVAL_NET_MODE", CFRB_NET_FP32);   // the reference evaluates a checkpoint with an fp32 forward
  auto model = torch::jit::load(model_path, torch::kCPU);
  RecursiveEvaluator ev(params, eval_device(), 8192);
  ev.setWeights(flat_weights_of(model));
  const auto strategy = ev.strategyRecursive();
  std::array<double, 2> e{};
  if (cfrb_exploitability(ev.handle(), strategy.data(), e.data()) < 0) throw std::runtime_error(cfrb_last_error());
  return (float)((e[0] + e[1]) / 2.0);
}

// compute_stats_with_net (pybind.cc:57-84): exploitability of compute_strategy_recursive_to_leaf with the net, and eval_net's MSE
// of the net against full-depth solves, with the beliefs defined by the net strategy and by the full-tree strategy.
std::tuple<float, float, float> compute_stats_with_net(RecursiveSolvingParams params, const std::string& model_path) {
  py::gil_scoped_release nogil;
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
    if (cfrb_exploitability(ev.handle(), net_strategy.data(), e.data()) < 0) throw std::runtime_error(cfrb_last_error());
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

// Synchronous helper for tests / benchmarks: run `waves` waves of a BatchedRlRunner on `device` and return all examples.
std::tuple<torch::Tensor, torch::Tensor> run_selfplay_waves(const RecursiveSolvingParams& cfg, int device, int seed, int waves,
                                                            py::object flat_weights) {
  std::vector<float> w;
  if (!flat_weights.is_none()) {
    auto t = flat_weights.cast<torch::Tensor>().to(torch::kCPU, torch::kFloat32).contiguous();
    w.assign(t.data_ptr<float>(), t.data_ptr<float>() + t.numel());
  }
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
py::dict recursive_eval_sampled(const RecursiveSolvingParams& cfg, int device, int num_repeats, int seed0, int batch_repeats,
                                int wave_capacity, py::object flat_weights) {
  std::vector<float> w;
  if (!flat_weights.is_none()) {
    auto t = flat_weights.cast<torch::Tensor>().to(torch::kCPU, torch::kFloat32).contiguous();
    w.assign(t.data_ptr<float>(), t.data_ptr<float>() + t.numel());
  }
  RecursiveEvalResult r;
  int A = 0, H = 0;
  {
    py::gil_scoped_release nogil;
    RecursiveEvaluator ev(cfg, device, wave_capacity);
    if (!w.empty()) ev.setWeights(w);
    r = ev.run(num_repeats, seed0, batch_repeats);
    A = ev.numActions(); H = ev.numHands();
  }
  const int64_t N = r.num_nodes;
  auto ss = torch::empty({N, H, A}), sr = torch::empty({N, H, 1}), fs = torch::empty({N, H, A});
  std::copy(r.summed_strategy.begin(), r.summed_strategy.end(), ss.data_ptr<float>());
  std::copy(r.summed_reach.begin(), r.summed_reach.end(), sr.data_ptr<float>());
  std::copy(r.final_strategy.begin(), r.final_strategy.end(), fs.data_ptr<float>());
  auto ex = torch::empty({(int64_t)r.exploitability.size(), 2}, torch::kFloat64);
  for (size_t i = 0; i < r.exploitability.size(); ++i) {
    ex[i][0] = r.exploitability[i][0];
    ex[i][1] = r.exploitability[i][1];
  }
  py::dict d;
  d["summed_strategy"] = ss; d["summed_reach"] = sr; d["final_strategy"] = fs;
  d["checkpoints"] = r.checkpoints; d["exploitability"] = ex; d["subgames_solved"] = r.subgames_solved; d["subgame_iters"] = r.subgame_iters;
  d["gpu_seconds"] = r.gpu_seconds;
  return d;
}

// compute_exploitability2 (subgame_solving.cc:802-816) of a dense full-tree strategy [N][H][A] on the GPU best-response kernel.
std::tuple<double, double> exploitability_of_strategy(int num_dice, int num_faces, torch::Tensor strategy) {
  auto s = strategy.to(torch::kCPU, torch::kFloat64).contiguous();
  cfrb_config c{};
  c.num_dice = num_dice; c.num_faces = num_faces; c.max_depth = 2; c.num_iters = 1; c.max_subgames = 1; c.device = eval_device();
  c.net_mode = CFRB_NET_ZERO; c.hidden = 256;
  cfrb_handle* h = nullptr;
  if (cfrb_create(&c, &h) < 0) throw std::runtime_error(std::string("cfrb_create: ") + cfrb_last_error());
  const int64_t A = cfrb_num_actions(h), H = cfrb_num_hands(h);
  const int64_t N = A <= 26 ? ((int64_t)1 << A) - 1 : -1;      // the full Liar's Dice tree has 2^A - 1 nodes
  std::array<double, 2> e{};
  int rc = -1;
  if (s.dim() == 3 && s.size(0) == N && s.size(1) == H && s.size(2) == A) rc = cfrb_exploitability(h, s.data_ptr<double>(), e.data());
  const std::string err = rc < 0 && s.dim() == 3 && s.size(0) == N ? cfrb_last_error() : "";
  cfrb_destroy(h);
  if (rc < 0) throw std::runtime_error(err.empty() ? "exploitability_of_strategy: strategy must be [num_full_tree_nodes, H, A]" : err);
  return std::make_tuple(e[0], e[1]);
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
      .def("update_priority", &ValuePrioritizedReplay::updatePriority);

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
  m.def("compute_stats_with_net", &compute_stats_with_net, py::arg("params"), py::arg("model_path"));
  m.def("create_cfr_thread", &create_cfr_thread, py::arg("model_locker"), py::arg("replay"), py::arg("cfg"), py::arg("seed"));
  m.def("run_selfplay_waves", &run_selfplay_waves, py::arg("cfg"), py::arg("device"), py::arg("seed"), py::arg("waves"),
        py::arg("flat_weights") = py::none(),
        "rebel_b200 extension: run `waves` waves of a BatchedRlRunner synchronously and return (queries, values).");
  m.def("exploitability_of_strategy", &exploitability_of_strategy, py::arg("num_dice"), py::arg("num_faces"), py::arg("strategy"),
        "rebel_b200 extension: compute_exploitability2 of a dense full-tree strategy (GPU best-response kernel).");
  m.def("recursive_eval_sampled", &recursive_eval_sampled, py::arg("cfg"), py::arg("device"), py::arg("num_repeats"), py::arg("seed") = 0,
        py::arg("batch_repeats") = 64, py::arg("wave_capacity") = 8192, py::arg("flat_weights") = py::none(),
        "rebel_b200 extension: the reference's `recursive_eval --cfr --num_repeats R` (sampled recursive strategies, float32 "
        "reach-weighted average, exploitability at powers of two) with the subgame solves batched on the GPU.");
}
