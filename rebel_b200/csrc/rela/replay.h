// Replay buffer of (value-net query, target values) rows — the consumer side of the data-generation path.
// Python surface identical to the reference's rela::ValuePrioritizedReplay (rela/pybind.cc:126-145,
// rela/prioritized_replay.h:224-506): same constructor, size / num_add / sample / pop_until / load / save / extract / push /
// update_priority, same blocking semantics (producers block while the ring of 1.25 x capacity rows is full, sampling
// evicts the oldest rows down to `capacity`), same on-disk record format (rela/types.cc:87-111).
//
// Not a port: the reference stores one pair of heap-allocated host tensors per example behind a vector of DataType and
// stacks a batch on the host before moving it to the training device (rela/types.cc:19-41).  Here the rows are DEVICE
// RESIDENT (SURVEY section 8 f-3): two [ring][dim] fp32 matrices in HBM behind the C ABI (cfrb_rows_*, include/cfrb200.h).
// Generator loops append a whole wave's examples with one device-to-device copy straight from the buffer their kernels wrote
// (addRowsDevice), and sample() gathers the batch on the device into the tensors it returns, on the consumer's own CUDA
// stream — an example never visits host memory between the kernel that produced it and the trainer's batch.  Only the
// bookkeeping the reference keeps under its mutex stays on the host: head / size, priorities, eviction marks, the sampler RNG.
// On a machine WITHOUT a CUDA device (the CPU test tier) the same class keeps the rows in host memory so that the ring /
// blocking / priority logic can be tested; nothing is computed there.
#pragma once
#include <c10/cuda/CUDAStream.h>
#include <torch/extension.h>

#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <functional>
#include <memory>
#include <mutex>
#include <random>
#include <sstream>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "../../../include/cfrb200.h"

namespace rela {

class ValueTransition {
 public:
  ValueTransition() = default;
  ValueTransition(const torch::Tensor& q, const torch::Tensor& v) : query(q), values(v) {}
  torch::Tensor query;
  torch::Tensor values;
};

// Where the rows of the ring live: HBM (cfrb_rows) when a CUDA device exists, host vectors otherwise.
class RowStore {
 public:
  RowStore() = default;
  RowStore(const RowStore&) = delete;
  RowStore& operator=(const RowStore&) = delete;
  ~RowStore() { if (dev_) cfrb_rows_destroy(dev_); }

  bool created() const { return q_dim_ >= 0; }
  bool onDevice() const { return dev_ != nullptr; }
  int device() const { return dev_ ? cfrb_rows_device(dev_) : -1; }
  int qDim() const { return q_dim_; }
  int vDim() const { return v_dim_; }

  void create(int64_t cap, int q_dim, int v_dim, int prefer_device) {
    cap_ = cap; q_dim_ = q_dim; v_dim_ = v_dim;
    const int ndev = cfrb_device_count();
    if (ndev > 0) {
      int d = prefer_device;
      if (const char* e = std::getenv("CFRB_REPLAY_DEVICE")) d = std::atoi(e);
      if (d < 0 || d >= ndev) d = 0;
      if (cfrb_rows_create(d, cap, q_dim, v_dim, &dev_) < 0) throw std::runtime_error(std::string("cfrb_rows_create: ") + cfrb_last_error());
    } else {
      hq_.assign((size_t)cap * q_dim, 0.f);
      hv_.assign((size_t)cap * v_dim, 0.f);
    }
  }
  // kind 0: host pointers, 1: device pointers on src_device
  void write(int64_t slot, int n, const float* q, const float* v, int kind, int src_device) {
    if (dev_) {
      if (cfrb_rows_write(dev_, slot, n, q, v, kind, src_device) < 0) throw std::runtime_error(std::string("cfrb_rows_write: ") + cfrb_last_error());
      return;
    }
    if (kind != 0) throw std::runtime_error("RowStore: device rows offered to a host-memory store");
    for (int i = 0; i < n; ++i) {
      const int64_t j = (slot + i) % cap_;
      std::copy(q + (size_t)i * q_dim_, q + (size_t)(i + 1) * q_dim_, hq_.begin() + (size_t)j * q_dim_);
      std::copy(v + (size_t)i * v_dim_, v + (size_t)(i + 1) * v_dim_, hv_.begin() + (size_t)j * v_dim_);
    }
  }
  void read(int64_t slot, int n, float* q, float* v) {
    if (dev_) {
      if (cfrb_rows_read(dev_, slot, n, q, v) < 0) throw std::runtime_error(std::string("cfrb_rows_read: ") + cfrb_last_error());
      return;
    }
    for (int i = 0; i < n; ++i) {
      const int64_t j = (slot + i) % cap_;
      std::copy(hq_.begin() + (size_t)j * q_dim_, hq_.begin() + (size_t)(j + 1) * q_dim_, q + (size_t)i * q_dim_);
      std::copy(hv_.begin() + (size_t)j * v_dim_, hv_.begin() + (size_t)(j + 1) * v_dim_, v + (size_t)i * v_dim_);
    }
  }
  // out_device: -1 host, else CUDA ordinal of out_q / out_v
  void gather(const std::vector<int>& ids, float* out_q, float* out_v, int out_device, void* stream) {
    if (dev_) {
      if (cfrb_rows_gather(dev_, ids.data(), (int)ids.size(), out_q, out_v, out_device, stream) < 0)
        throw std::runtime_error(std::string("cfrb_rows_gather: ") + cfrb_last_error());
      return;
    }
    if (out_device >= 0) throw std::runtime_error("RowStore: no CUDA device");
    for (size_t i = 0; i < ids.size(); ++i) {
      const int64_t j = ids[i];
      std::copy(hq_.begin() + (size_t)j * q_dim_, hq_.begin() + (size_t)(j + 1) * q_dim_, out_q + i * q_dim_);
      std::copy(hv_.begin() + (size_t)j * v_dim_, hv_.begin() + (size_t)(j + 1) * v_dim_, out_v + i * v_dim_);
    }
  }

 private:
  cfrb_rows* dev_ = nullptr;
  std::vector<float> hq_, hv_;
  int64_t cap_ = 0;
  int q_dim_ = -1, v_dim_ = -1;
};

class ValuePrioritizedReplay {
 public:
  ValuePrioritizedReplay(int capacity, int seed, float alpha, float beta, int prefetch, bool use_priority, bool compressed_values)
      : alpha_(alpha), beta_(beta), prefetch_(prefetch), capacity_(capacity), ring_(int(1.25 * capacity)), seed_(seed),
        use_priority_(use_priority), weights_(ring_, 0.f), evicted_(ring_, 0) {
    if (compressed_values) throw std::runtime_error("ValuePrioritizedReplay: compressed_values is not supported by rebel_b200");
    if (capacity <= 0) throw std::runtime_error("ValuePrioritizedReplay: capacity must be positive");
    rng_.seed(seed);
  }

  int size() const { std::lock_guard<std::mutex> lk(m_); return size_; }
  int numAdd() const { return num_add_.load(); }
  // rebel_b200 extension: CUDA ordinal the rows live on (-1: host memory, no CUDA device; -2: nothing stored yet)
  int storageDevice() const { std::lock_guard<std::mutex> lk(m_); return store_.created() ? store_.device() : -2; }

  // Producer paths.  n rows of width q_dim / v_dim; priority may be null (= 1).  Blocks while the ring is full
  // (ConcurrentQueue::blockAppend, prioritized_replay.h:59-96); `cancelled` (optional) is polled whenever the buffer is woken
  // (wake()) so that a terminating generator loop can leave — it returns false then, without closing the buffer for others.
  bool addRows(const float* q, int q_dim, const float* v, int v_dim, int n, const float* priority,
               const std::function<bool()>& cancelled = nullptr) {
    return append(q, q_dim, v, v_dim, n, priority, /*kind=*/0, /*src_device=*/-1, cancelled);
  }
  // The same for rows that already live in device memory (a generator's example buffer): one device-to-device copy.
  bool addRowsDevice(const float* dev_q, int q_dim, const float* dev_v, int v_dim, int n, int src_device,
                     const std::function<bool()>& cancelled = nullptr) {
    return append(dev_q, q_dim, dev_v, v_dim, n, nullptr, /*kind=*/1, src_device, cancelled);
  }
  void wake() { cv_space_.notify_all(); }

  // add(batch, priority) of the reference: slices an [n, ...] transition into rows (prioritized_replay.h:254-261)
  void add(const ValueTransition& batch, const torch::Tensor& priority) {
    auto p = priority.to(torch::kCPU, torch::kFloat32).contiguous();
    const int n = (int)p.size(0);
    auto q = batch.query, v = batch.values;
    if (q.dim() == 1) q = q.unsqueeze(0);
    if (v.dim() == 1) v = v.unsqueeze(0);
    if (q.size(0) != n || v.size(0) != n) throw std::runtime_error("ValuePrioritizedReplay.add: batch/priority size mismatch");
    if (q.is_cuda() && v.is_cuda() && q.get_device() == v.get_device() && cfrb_device_count() > 0) {
      // rows that are already on a GPU stay there
      q = q.to(torch::kFloat32).contiguous(); v = v.to(torch::kFloat32).contiguous();
      c10::cuda::getCurrentCUDAStream(q.get_device()).synchronize();
      append(q.data_ptr<float>(), (int)q.size(1), v.data_ptr<float>(), (int)v.size(1), n, p.data_ptr<float>(), 1, (int)q.get_device(), nullptr);
      return;
    }
    q = q.to(torch::kCPU, torch::kFloat32).contiguous();
    v = v.to(torch::kCPU, torch::kFloat32).contiguous();
    addRows(q.data_ptr<float>(), (int)q.size(1), v.data_ptr<float>(), (int)v.size(1), n, p.data_ptr<float>());
  }

  std::tuple<ValueTransition, torch::Tensor> sample(int batchsize, const std::string& device) {
    if (!sampled_ids_.empty() && use_priority_)
      throw std::runtime_error("ValuePrioritizedReplay.sample: previous samples' priority has not been updated");
    std::unique_lock<std::mutex> lk(m_);
    if (size_ <= 0) throw std::runtime_error("ValuePrioritizedReplay.sample: buffer is empty");
    auto w = torch::zeros({batchsize}, torch::kFloat32);
    float* wp = w.data_ptr<float>();
    std::vector<int> ids(batchsize);
    const int size = size_;
    const double sum = sum_;
    if (!use_priority_) {   // sample_no_priorities_ (prioritized_replay.h:451-486)
      std::uniform_int_distribution<> dist(0, size - 1);
      for (int i = 0; i < batchsize; ++i) {
        const int j = (head_ + dist(rng_)) % ring_;
        ids[i] = j; wp[i] = weights_[j]; evicted_[j] = 0;
      }
    } else {                // stratified proportional sampling (prioritized_replay.h:373-449)
      const float segment = (float)sum / batchsize;
      std::uniform_real_distribution<float> dist(0.0f, segment);
      double acc = 0; int next = 0, id = head_; float wj = 0;
      for (int i = 0; i < batchsize; ++i) {
        float r = std::min((float)sum - 0.1f, dist(rng_) + i * segment);
        while (next < size && !(acc > 0 && acc >= r)) {
          id = (head_ + next) % ring_; wj = weights_[id]; acc += wj; ++next;
        }
        ids[i] = id; wp[i] = wj; evicted_[id] = 0;
      }
    }
    // makeBatch (rela/types.cc:19-41): gather the rows into the batch tensors — on the device when the rows are there
    const bool to_gpu = device != "cpu";
    ValueTransition batch;
    if (store_.onDevice() && to_gpu) {
      const auto d = torch::Device(device);
      const int di = d.has_index() ? d.index() : 0;
      auto opts = torch::TensorOptions().dtype(torch::kFloat32).device(torch::Device(torch::kCUDA, di));
      batch.query = torch::empty({batchsize, store_.qDim()}, opts);
      batch.values = torch::empty({batchsize, store_.vDim()}, opts);
      store_.gather(ids, batch.query.data_ptr<float>(), batch.values.data_ptr<float>(), di, (void*)c10::cuda::getCurrentCUDAStream(di).stream());
    } else {
      auto opts = torch::TensorOptions().dtype(torch::kFloat32).pinned_memory(to_gpu && cfrb_device_count() > 0);
      batch.query = torch::empty({batchsize, store_.qDim()}, opts);
      batch.values = torch::empty({batchsize, store_.vDim()}, opts);
      store_.gather(ids, batch.query.data_ptr<float>(), batch.values.data_ptr<float>(), -1, nullptr);
      if (to_gpu) {
        const auto d = torch::Device(device);
        batch.query = batch.query.to(d, /*non_blocking=*/true);
        batch.values = batch.values.to(d, /*non_blocking=*/true);
      }
    }
    if (size_ > capacity_) popLocked(size_ - capacity_);   // evict oldest down to capacity (prioritized_replay.h:474-477)
    lk.unlock();
    sampled_ids_ = ids;
    if (use_priority_) {
      w = torch::pow(size * (w / (float)sum), -beta_);
      w /= w.max();
    }
    if (to_gpu) w = w.to(torch::Device(device));
    return std::make_tuple(batch, w);
  }

  void updatePriority(const torch::Tensor& priority) {
    if (priority.size(0) == 0) { sampled_ids_.clear(); return; }
    if ((int)sampled_ids_.size() != priority.size(0)) throw std::runtime_error("update_priority: size mismatch");
    auto p = torch::pow(priority.to(torch::kCPU, torch::kFloat32), alpha_).contiguous();
    const float* pp = p.data_ptr<float>();
    std::lock_guard<std::mutex> lk(m_);
    for (size_t i = 0; i < sampled_ids_.size(); ++i) {   // ConcurrentQueue::update (prioritized_replay.h:132-150): evicted rows are skipped
      const int id = sampled_ids_[i];
      if (evicted_[id]) continue;
      sum_ += pp[i] - weights_[id];
      weights_[id] = pp[i];
    }
    sampled_ids_.clear();
  }

  void popUntil(int new_size) {
    std::lock_guard<std::mutex> lk(m_);
    if (size_ > new_size) popLocked(size_ - new_size);
  }

  // Flat binary records: int32 qsize, int32 vsize, float[q], float[v] (rela/types.cc:87-111)
  void save(const std::string& path) {
    std::lock_guard<std::mutex> lk(m_);
    FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) throw std::runtime_error("cannot open " + path);
    if (size_ > 0) {
      const int qd = store_.qDim(), vd = store_.vDim();
      std::vector<float> q((size_t)size_ * qd), v((size_t)size_ * vd);
      store_.read(head_, size_, q.data(), v.data());
      for (int i = 0; i < size_; ++i) {
        std::fwrite(&qd, sizeof(int), 1, f); std::fwrite(&vd, sizeof(int), 1, f);
        std::fwrite(&q[(size_t)i * qd], sizeof(float), qd, f);
        std::fwrite(&v[(size_t)i * vd], sizeof(float), vd, f);
      }
    }
    std::fclose(f);
  }

  void load(const std::string& path, float priority, int max_size, int stride) {
    FILE* f = std::fopen(path.c_str(), "rb");
    if (!f) throw std::runtime_error("cannot open " + path);
    std::vector<float> q, v, bq, bv, bp;
    int qd = 0, vd = 0;
    auto flush = [&]() {
      if (!bp.empty()) addRows(bq.data(), qd, bv.data(), vd, (int)bp.size(), bp.data());
      bq.clear(); bv.clear(); bp.clear();
    };
    for (int added = 0, i = 0;; ++i) {
      if (max_size > 0 && added == max_size) break;
      int qs = 0, vs = 0;
      if (std::fread(&qs, sizeof(int), 1, f) != 1 || std::fread(&vs, sizeof(int), 1, f) != 1) break;
      q.resize(qs); v.resize(vs);
      if ((int)std::fread(q.data(), sizeof(float), qs, f) != qs || (int)std::fread(v.data(), sizeof(float), vs, f) != vs) break;
      if (stride > 1 && i % stride != 0) continue;
      if (!bp.empty() && (qs != qd || vs != vd)) flush();
      qd = qs; vd = vs;
      bq.insert(bq.end(), q.begin(), q.end()); bv.insert(bv.end(), v.begin(), v.end()); bp.push_back(priority);
      if ((int)bp.size() >= 4096) flush();     // one host-to-device copy per block, not per record
      ++added;
    }
    flush();
    std::fclose(f);
  }

  // rebel_b200 extension: the whole observable state, so that a stopped training run continues bit for bit.  Binary file: a
  // header (magic, format version, the constructor parameters, row widths, size, num_add, sum), the sampler's mt19937 state as
  // text, then the live rows in order from head: weights [n] and rows (query, values) in blocks.  Host byte order.
  void saveState(const std::string& path) {
    std::lock_guard<std::mutex> lk(m_);
    if (use_priority_ && !sampled_ids_.empty())
      throw std::runtime_error("ValuePrioritizedReplay.save_state: the priorities of the last sample have not been updated");
    FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) throw std::runtime_error("ValuePrioritizedReplay.save_state: cannot open " + path);
    StateHeader hd = header();
    hd.q_dim = store_.created() ? store_.qDim() : -1;
    hd.v_dim = store_.created() ? store_.vDim() : -1;
    hd.size = size_; hd.num_add = num_add_.load(); hd.sum = sum_;
    std::ostringstream os;
    os << rng_;
    const std::string rng = os.str();
    hd.rng_bytes = (int32_t)rng.size();
    bool ok = std::fwrite(&hd, sizeof hd, 1, f) == 1 && std::fwrite(rng.data(), 1, rng.size(), f) == rng.size();
    std::vector<float> w(size_);
    for (int i = 0; i < size_; ++i) w[i] = weights_[(head_ + i) % ring_];
    ok = ok && (int)std::fwrite(w.data(), sizeof(float), size_, f) == size_;
    std::vector<float> q, v;
    for (int i = 0; ok && i < size_; i += kStateBlock) {
      const int n = std::min(kStateBlock, size_ - i);
      q.resize((size_t)n * hd.q_dim); v.resize((size_t)n * hd.v_dim);
      store_.read((head_ + i) % ring_, n, q.data(), v.data());
      ok = std::fwrite(q.data(), sizeof(float), q.size(), f) == q.size() && std::fwrite(v.data(), sizeof(float), v.size(), f) == v.size();
    }
    ok = std::fclose(f) == 0 && ok;
    if (!ok) throw std::runtime_error("ValuePrioritizedReplay.save_state: write to " + path + " failed");
  }

  // Restores saveState's file into this buffer, which must be empty (nothing ever added) and built with the same parameters.  The
  // rows are laid out from slot 0; sample(), size(), num_add(), eviction and producer blocking behave as in the saved buffer.
  // prefer_device: the CUDA ordinal of the rows when a device exists (CFRB_REPLAY_DEVICE overrides it, as for a first append).
  void loadState(const std::string& path, int prefer_device) {
    std::lock_guard<std::mutex> lk(m_);
    const std::string who = "ValuePrioritizedReplay.load_state(" + path + "): ";
    if (num_add_.load() != 0 || store_.created()) throw std::runtime_error(who + "the buffer is not empty");
    FILE* f = std::fopen(path.c_str(), "rb");
    if (!f) throw std::runtime_error(who + "cannot open the file");
    std::unique_ptr<FILE, int (*)(FILE*)> closer(f, std::fclose);
    StateHeader hd{};
    if (std::fread(&hd, sizeof hd, 1, f) != 1) throw std::runtime_error(who + "truncated header");
    const StateHeader want = header();
    if (hd.magic != want.magic) throw std::runtime_error(who + "not a replay state file");
    if (hd.version != want.version) throw std::runtime_error(who + "format version " + std::to_string(hd.version) + ", expected " + std::to_string(want.version));
    auto differs = [&](const char* name, double got, double exp) {
      return std::runtime_error(who + name + " is " + std::to_string(got) + " in the file and " + std::to_string(exp) + " in this buffer");
    };
    if (hd.capacity != want.capacity) throw differs("capacity", hd.capacity, want.capacity);
    if (hd.seed != want.seed) throw differs("seed", hd.seed, want.seed);
    if (hd.alpha != want.alpha) throw differs("alpha", hd.alpha, want.alpha);
    if (hd.beta != want.beta) throw differs("beta", hd.beta, want.beta);
    if (hd.prefetch != want.prefetch) throw differs("prefetch", hd.prefetch, want.prefetch);
    if (hd.use_priority != want.use_priority) throw differs("use_priority", hd.use_priority, want.use_priority);
    if (hd.size < 0 || hd.size > ring_ || hd.num_add < hd.size || hd.rng_bytes <= 0 || hd.rng_bytes > (1 << 16) ||
        (hd.size > 0 && (hd.q_dim <= 0 || hd.v_dim <= 0)))
      throw std::runtime_error(who + "inconsistent header");
    std::string rng(hd.rng_bytes, '\0');
    if (std::fread(rng.data(), 1, rng.size(), f) != rng.size()) throw std::runtime_error(who + "truncated sampler state");
    std::mt19937 gen;
    std::istringstream is(rng);
    if (!(is >> gen)) throw std::runtime_error(who + "bad sampler state");
    std::vector<float> w(hd.size);
    if ((int)std::fread(w.data(), sizeof(float), hd.size, f) != hd.size) throw std::runtime_error(who + "truncated weights");
    // read every row before the store exists, so that a truncated file leaves the buffer empty
    std::vector<float> q((size_t)hd.size * std::max(hd.q_dim, 0)), v((size_t)hd.size * std::max(hd.v_dim, 0));
    for (int i = 0; i < hd.size; i += kStateBlock) {
      const int n = std::min(kStateBlock, hd.size - i);
      if (std::fread(q.data() + (size_t)i * hd.q_dim, sizeof(float), (size_t)n * hd.q_dim, f) != (size_t)n * hd.q_dim ||
          std::fread(v.data() + (size_t)i * hd.v_dim, sizeof(float), (size_t)n * hd.v_dim, f) != (size_t)n * hd.v_dim)
        throw std::runtime_error(who + "truncated rows");
    }
    if (std::fgetc(f) != EOF) throw std::runtime_error(who + "trailing bytes after the rows");
    if (hd.q_dim > 0) {
      store_.create(ring_, hd.q_dim, hd.v_dim, prefer_device);
      if (hd.size > 0) store_.write(0, hd.size, q.data(), v.data(), /*kind=*/0, -1);
    }
    std::copy(w.begin(), w.end(), weights_.begin());
    std::fill(evicted_.begin(), evicted_.end(), 0);
    head_ = 0; size_ = hd.size; sum_ = hd.sum; num_add_ = hd.num_add;
    rng_ = gen;
    sampled_ids_.clear();
  }

  // Whole content as [queries [n,Q], values [n,H], weights [n]] and empty the buffer (prioritized_replay.h:338-345)
  std::vector<torch::Tensor> extract() {
    std::lock_guard<std::mutex> lk(m_);
    const int n = size_;
    const int qd = std::max(store_.qDim(), 0), vd = std::max(store_.vDim(), 0);
    auto q = torch::empty({n, qd}), v = torch::empty({n, vd}), w = torch::empty({n});
    if (n > 0) store_.read(head_, n, q.data_ptr<float>(), v.data_ptr<float>());
    for (int i = 0; i < n; ++i) w.data_ptr<float>()[i] = std::pow(weights_[(head_ + i) % ring_], 1.f / alpha_);   // :341
    popLocked(n);
    return {q, v, w};
  }

  void push(std::vector<torch::Tensor> data) {
    if (data.size() != 3) throw std::runtime_error("push expects [queries, values, weights]");
    add(ValueTransition(data[0], data[1]), data[2]);
  }

 private:
  struct StateHeader {
    uint32_t magic, version;
    int32_t capacity, seed, prefetch, use_priority;
    float alpha, beta;
    int32_t q_dim, v_dim, size, num_add;
    double sum;
    int32_t rng_bytes, pad;
  };
  static constexpr int kStateBlock = 65536;   // rows per host <-> store copy of save_state / load_state
  StateHeader header() const {
    StateHeader hd{};
    hd.magic = 0x53525052u;   // "RPRS"
    hd.version = 1;
    hd.capacity = capacity_; hd.seed = seed_; hd.prefetch = prefetch_; hd.use_priority = use_priority_ ? 1 : 0;
    hd.alpha = alpha_; hd.beta = beta_;
    return hd;
  }

  bool append(const float* q, int q_dim, const float* v, int v_dim, int n, const float* priority, int kind, int src_device,
              const std::function<bool()>& cancelled) {
    if (n <= 0) return true;
    std::unique_lock<std::mutex> lk(m_);
    if (!store_.created()) store_.create(ring_, q_dim, v_dim, kind == 1 ? src_device : 0);
    else if (q_dim != store_.qDim() || v_dim != store_.vDim()) throw std::runtime_error("ValuePrioritizedReplay: row width changed");
    if (n > ring_) throw std::runtime_error("ValuePrioritizedReplay: block larger than the buffer");
    cv_space_.wait(lk, [&] { return size_ + n <= ring_ || (cancelled && cancelled()); });
    if (size_ + n > ring_) return false;   // cancelled while waiting
    const int first = (head_ + size_) % ring_;
    if (kind == 1 && !store_.onDevice()) throw std::runtime_error("ValuePrioritizedReplay: device rows without a CUDA device");
    store_.write(first, n, q, v, kind, src_device);
    double add = 0;
    for (int i = 0; i < n; ++i) {
      const int j = (first + i) % ring_;
      float w = priority ? priority[i] : 1.f;
      if (use_priority_) w = std::pow(w, alpha_);
      weights_[j] = w;                       // evicted_[j] is NOT reset here (blockAppend never touches it, :59-96)
      add += w;
    }
    size_ += n;
    sum_ += add;
    num_add_ += n;
    return true;
  }
  void popLocked(int n) {
    for (int i = 0; i < n; ++i) {
      sum_ -= weights_[head_];
      evicted_[head_] = 1;
      head_ = (head_ + 1) % ring_;
    }
    size_ -= n;
    cv_space_.notify_all();
  }

  const float alpha_, beta_;
  const int prefetch_, capacity_, ring_, seed_;
  const bool use_priority_;
  mutable std::mutex m_;
  std::condition_variable cv_space_;
  RowStore store_;
  std::vector<float> weights_;
  std::vector<char> evicted_;
  int head_ = 0, size_ = 0;
  double sum_ = 0;
  std::atomic<int> num_add_{0};
  std::vector<int> sampled_ids_;
  std::mt19937 rng_;
};

}  // namespace rela
