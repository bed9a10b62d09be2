// Device-resident self-play walk: RlRunner::step (recursive_solving.cc:160-275) for K games in lock-step, one thread per game.
//
// The reference plays ONE game per CPU thread: solve the subgame at the current public state, at iteration `act_iteration`
// sample the next state with the solver's sampling strategy (sample_state_to_leaf :192-246 / sample_state_single :248-275),
// Bayes-update the beliefs, and emit two training examples per solved subgame (subgame_solving.cc:672-676).  Here a *wave*
// solves the current subgame of every game at once (cfr_iter kernels + value net); these kernels do everything in between two
// waves ON THE DEVICE, so a self-play loop never brings strategies, beliefs or examples to the host:
//
//   sp_examples   two (query, target) rows per finished subgame, straight into a device buffer (the replay's ring)
//   sp_advance    per game: br_sampler / eps / hand / action draws, sampling-belief and real-belief updates with
//                 eps-normalisation, next public state (or a fresh game after a terminal state)
//   sp_begin      per game: act_iteration ~ U{0..num_iters} and the descriptor of its next subgame (template, player, beliefs)
//   sp_scan       prefix sum of the pseudo-leaf counts -> packed value-net row offsets, wave size, total rows; the CFR
//                 kernel's schedule (wave positions, costliest template first)
//   sp_share      after the last iteration: the results of the wave's one initial-state solve to every game that shares it
//
// Every game owns a std::mt19937 stream (state words interleaved [624][K] so that the threads of a warp touch consecutive
// addresses) and the libstdc++ distributions the reference uses are restated bit for bit (uniform_int_distribution = Lemire's
// nearly-divisionless method, generate_canonical<float,24> / <double,53>, discrete_distribution = normalise + partial sums +
// lower_bound), with the reference's draw ORDER and fp64 belief arithmetic (this header is compiled into the -fmad=false
// translation unit).  Game g of a runner seeded with s therefore replays the reference's RlRunner(seed = seeds[g]) exactly,
// as long as the solver's strategies agree — which the tests check against the compiled reference with the zero net.
#pragma once
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include "cfr_tree.h"
#include "cfr_types.h"

namespace cfrb {

// ---------------------------------------------------------------- std::mt19937, state word i of game g at mt[i * K + g]
struct SpRng {
  uint32_t* s; int K; int idx;
  __device__ __forceinline__ uint32_t& w(int i) { return s[(size_t)i * K]; }
  __device__ uint32_t next() {
    if (idx >= 624) {
      for (int i = 0; i < 624; ++i) {
        const uint32_t y = (w(i) & 0x80000000u) | (w(i + 1 < 624 ? i + 1 : 0) & 0x7fffffffu);
        const int j = i + 397 < 624 ? i + 397 : i + 397 - 624;
        w(i) = w(j) ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
      }
      idx = 0;
    }
    uint32_t y = w(idx++);
    y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
    return y;
  }
  // std::uniform_int_distribution<int>(a, b) on a 32-bit generator (bits/uniform_int_dist.h, _S_nd)
  __device__ int uniform_int(int a, int b) {
    const uint32_t urange = (uint32_t)b - (uint32_t)a;
    if (urange == 0xffffffffu) return (int)(next() + (uint32_t)a);
    const uint32_t range = urange + 1;
    uint64_t product = (uint64_t)next() * (uint64_t)range;
    uint32_t low = (uint32_t)product;
    if (low < range) {
      const uint32_t threshold = (uint32_t)(0u - range) % range;
      while (low < threshold) { product = (uint64_t)next() * (uint64_t)range; low = (uint32_t)product; }
    }
    return (int)((uint32_t)(product >> 32) + (uint32_t)a);
  }
  // std::generate_canonical<float, 24>: one draw
  __device__ float canonical_f() {
    const float r = (float)next() / 4294967296.0f;
    return r >= 1.0f ? 0.99999994f : r;            // nextafterf(1, 0)
  }
  // std::generate_canonical<double, 53>: two draws
  __device__ double canonical_d() {
    double sum = (double)next();
    sum += (double)next() * 4294967296.0;
    const double r = sum / 18446744073709551616.0;
    return r >= 1.0 ? 0.99999999999999989 : r;     // nextafter(1, 0)
  }
};

// std::mt19937(x) into an interleaved state whose words lie `stride` apart (word i at st[i * stride])
__device__ __forceinline__ void mt_seed_strided(uint32_t* st, int stride, uint32_t x) {
  st[0] = x;
  for (int i = 1; i < 624; ++i) { x = 1812433253u * (x ^ (x >> 30)) + (uint32_t)i; st[(size_t)i * stride] = x; }
}

// std::discrete_distribution<int> over n weights w(0..n-1): probabilities w/sum, partial sums, last one forced to 1,
// lower_bound of a canonical double.  (The linear scan returns the same index as the binary search: the sums never decrease.)
template <typename W>
__device__ int sp_discrete(SpRng& rng, int n, W w) {
  if (n < 2) return 0;
  double sum = 0;
  for (int i = 0; i < n; ++i) sum += w(i);
  const double p = rng.canonical_d();
  double acc = 0;
  for (int i = 0; i < n - 1; ++i) {
    acc += w(i) / sum;
    if (!(acc < p)) return i;
  }
  return n - 1;
}

// The act_iteration of a sampled policy's subgame (compute_sampled_strategy_recursive_to_leaf, recursive_solving.cc:304-319):
// weight i / 2 + 1 on even i < n, 0 on odd i.
__device__ __forceinline__ int sp_act_iteration(SpRng& rng, int n) {
  return sp_discrete(rng, n, [](int i) { return i % 2 ? 0.0 : (i / 2. + 1); });
}

// normalize_beliefs_inplace (recursive_solving.cc:41-44 -> normalize_probabilities_safe, util.h:68-78)
__device__ __forceinline__ void sp_normalize(double* b, int H) {
  double s = 0;
  for (int h = 0; h < H; ++h) s += b[h] + 1e-80;
  for (int h = 0; h < H; ++h) b[h] = (b[h] + 1e-80) / s;
}

// The average strategy an agent acts with, for one (node, hand) of a solved subgame's table T: child j of the node is entry
// T[(r0 + j) * H + h], r0 = the node's first child - 1 and h the hand.  FP's average and the sampled snapshot are used as they are
// (normalise false); CFR's sum is divided by its serial fp64 sum over the node's nc children, and is uniform while the acting
// player has no update yet (untouched) or when that sum is not positive (cfrb_fetch_compact kind 4, normalise_avg in cfrb_api.cu).
// Every play and exploitability walk reads average strategies through these, so they all agree bit for bit.
template <typename real>
__device__ __forceinline__ double avg_row_sum(const real* T, int r0, int h, int H, int nc) {
  double sum = 0;
  for (int j = 0; j < nc; ++j) sum += (double)T[(size_t)(r0 + j) * H + h];
  return sum;
}
__device__ __forceinline__ double avg_entry(double v, double sum, int nc, bool normalise, bool untouched) {
  return !normalise ? v : (sum > 0 && !untouched) ? v / sum : 1.0 / nc;
}
// child j alone
template <typename real>
__device__ __forceinline__ double avg_prob(const real* T, int r0, int h, int H, int nc, bool normalise, bool untouched, int j) {
  const double v = (double)T[(size_t)(r0 + j) * H + h];
  if (!normalise || untouched) return avg_entry(v, 0.0, nc, normalise, untouched);
  return avg_entry(v, avg_row_sum(T, r0, h, H, nc), nc, true, false);
}
// every child, into out[j * H]
template <typename real>
__device__ __forceinline__ void avg_row(double* out, const real* T, int r0, int h, int H, int nc, bool normalise, bool untouched) {
  const double sum = normalise ? avg_row_sum(T, r0, h, H, nc) : 0.0;
  for (int j = 0; j < nc; ++j) out[j * H] = avg_entry((double)T[(size_t)(r0 + j) * H + h], sum, nc, normalise, untouched);
}

__global__ void __launch_bounds__(128) sp_seed_kernel(SpDev p, const uint32_t* __restrict__ seeds) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.K) return;
  mt_seed_strided(p.mt + g, p.K, seeds[g]);
  p.mt_idx[g] = 624;
  p.g_last_bid[g] = -1; p.g_player[g] = 0;                       // RlRunner::step :161-163
  for (int i = 0; i < 2 * p.H; ++i) p.g_beliefs[(size_t)g * 2 * p.H + i] = 1.0 / p.H;
}

// First half of RlRunner::step's loop body for every game: the act_iteration draw (:168-169) and the subgame descriptor.
template <typename real>
__global__ void __launch_bounds__(128) sp_begin_kernel(SpDev p, real* __restrict__ wave_beliefs) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.K) return;
  SpRng rng{p.mt + g, p.K, p.mt_idx[g]};
  p.sg_act[g] = rng.uniform_int(0, p.iters);
  p.mt_idx[g] = rng.idx;
  p.sg_tmpl[g] = p.g_last_bid[g] + 1;
  p.sg_player[g] = p.g_player[g];
  // The initial state (sp_seed_kernel, the terminal reset of sp_advance_kernel), told by the belief bits: a game whose beliefs only
  // compare equal to 1 / H (an imported session) is solved on its own
  const double* gb = p.g_beliefs + (size_t)g * 2 * p.H;
  const long long uniform = __double_as_longlong(1.0 / p.H);
  bool init = p.g_last_bid[g] == -1 && p.g_player[g] == 0;
  for (int i = 0; i < 2 * p.H; ++i) {
    wave_beliefs[(size_t)g * 2 * p.H + i] = (real)gb[i];
    init = init && __double_as_longlong(gb[i]) == uniform;
  }
  if (p.share) p.sg_init[g] = init;
}

// Inclusive sums of a thread's V values over the 1024 threads of the CTA, through part[V * 1024]: x[i] becomes the sum of x[i]
// over threads 0 .. threadIdx.x, so thread 1023 holds the totals (and so does part[i * 1024 + 1023]).
template <int V>
__device__ void sp_block_scan(int* part, int (&x)[V]) {
  const int t = threadIdx.x;
  __syncthreads();                               // earlier readers of part[] are done
  for (int i = 0; i < V; ++i) part[i * 1024 + t] = x[i];
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    int u[V];
    for (int i = 0; i < V; ++i) u[i] = t >= d ? part[i * 1024 + t - d] : 0;
    __syncthreads();
    for (int i = 0; i < V; ++i) part[i * 1024 + t] += u[i];
    __syncthreads();
  }
  for (int i = 0; i < V; ++i) x[i] = part[i * 1024 + t];
}
__device__ __forceinline__ int sp_block_scan(int* part, int x) {
  int v[1] = {x};
  sp_block_scan(part, v);
  return v[0];
}

// Exclusive prefix sum of the pseudo-leaf counts of the wave's subgames (one CTA; K is at most a few 10^4).
__global__ void __launch_bounds__(1024) sp_scan_kernel(SpDev p) {
  __shared__ int part[1024];
  const int t = threadIdx.x, per = (p.K + 1023) / 1024;
  const int b = t * per, e = min(p.K, b + per);
  int s = 0;
  for (int g = b; g < e; ++g) s += p.tmpl[p.sg_tmpl[g]].L;
  const int rows = sp_block_scan(part, s);
  int off = rows - s;
  for (int g = b; g < e; ++g) { p.sg_row_off[g] = off; off += p.tmpl[p.sg_tmpl[g]].L; }
  if (t == 1023) { p.wave[0] = p.K; p.wave[1] = rows; }
  // The CFR kernel's schedule: the wave positions in template-rank order, a stable counting sort (schedule_order, cfr_tree.h)
  // with one block-wide exclusive scan of the per-thread counts per rank.  part[] is reused for the 32 warp totals.
  const int lane = t & 31, warp = t >> 5;
  int base = 0;
  for (int r = 0; r < p.A; ++r) {
    int c = 0;
    for (int g = b; g < e; ++g) c += p.tmpl_rank[p.sg_tmpl[g]] == r;
    int x = c;                                   // inclusive scan within the warp
    for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    __syncthreads();                             // the previous rank's reads of part[] are done
    if (lane == 31) part[warp] = x;
    __syncthreads();
    int wsum = part[lane];                       // inclusive scan of the warp totals, in every warp
    for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, wsum, d); if (lane >= d) wsum += y; }
    const int before = __shfl_sync(0xffffffffu, wsum, (warp + 31) & 31);
    int pos = base + (warp ? before : 0) + x - c;
    for (int g = b; g < e; ++g)
      if (p.tmpl_rank[p.sg_tmpl[g]] == r) p.sg_order[pos++] = g;
    base += __shfl_sync(0xffffffffu, wsum, 31);
  }
  // Every initial-state subgame solves the same thing bit for bit (its template, player and beliefs are the same, and so are the
  // weights and num_iters), so a shared wave solves only the lowest one, the representative; the solved set -- every game but the
  // copies -- keeps the schedule's order in sg_order[solved_off ..].  Every game keeps its rows, so that a rerun of the whole wave
  // (materialise_sum) finds them; a copy's rows are simply never written.
  int n_solved = p.K, solved_at = 0;             // the solved set: sg_order[solved_at, solved_at + n_solved)
  if (!p.share) {
    if (t == 1023) { p.wave[2] = p.K; p.wave[3] = -1; }
  } else {
    __shared__ int rep_s;
    if (t == 0) rep_s = INT_MAX;
    int first = INT_MAX;
    for (int g = e - 1; g >= b; --g) if (p.sg_init[g]) first = g;
    __syncthreads();                               // rep_s is set, and the schedule above is visible to the whole CTA
    if (first != INT_MAX) atomicMin(&rep_s, first);
    __syncthreads();
    const int rep = rep_s == INT_MAX ? -1 : rep_s;
    auto solved = [&](int g) { return !p.sg_init[g] || g == rep; };
    int c = 0;
    for (int i = b; i < e; ++i) c += solved(p.sg_order[i]);
    n_solved = sp_block_scan(part, c);
    int pos = n_solved - c;
    for (int i = b; i < e; ++i)
      if (solved(p.sg_order[i])) p.sg_order[p.solved_off + pos++] = p.sg_order[i];
    if (t == 1023) { p.wave[2] = n_solved; p.wave[3] = rep; }
    n_solved = part[1023];
    solved_at = p.solved_off;
  }
  // The CFR kernel's wide tickets (wide_count, cfr_tree.h) from the solved set's costs, in p.wave[4]
  __shared__ unsigned long long wide_s[2];         // summed cost, subgames with at least kWideShare of the costliest template's
  if (t == 0) { wide_s[0] = 0; wide_s[1] = 0; }
  long long max_cost = 0;
  for (int r = 0; r < p.A; ++r) max_cost = max(max_cost, (long long)template_cost(p.tmpl[r].N, p.tmpl[r].L, p.H));
  __syncthreads();                                 // wide_s is set, and the solved set is visible to the whole CTA
  const int per_s = (n_solved + 1023) / 1024, sb = t * per_s, se = min(n_solved, sb + per_s);
  unsigned long long tot = 0, big = 0;
  for (int i = sb; i < se; ++i) {
    const int g = p.sg_order[solved_at + i];
    const long long cost = template_cost(p.tmpl[p.sg_tmpl[g]].N, p.tmpl[p.sg_tmpl[g]].L, p.H);
    tot += cost;
    big += (double)cost >= kWideShare * (double)max_cost;
  }
  if (tot) atomicAdd(&wide_s[0], tot);
  if (big) atomicAdd(&wide_s[1], big);
  __syncthreads();
  const int warps = min(p.wide_warps, 4 * ((p.K + 3) / 4));   // a launch has at most ceil(K / 4) CTAs (launch_iter)
  if (t == 0) p.wave[4] = wide_count((int64_t)wide_s[1], (int64_t)wide_s[0], max_cost, n_solved, warps, p.wide_force);
}

// The copies of a shared wave (sp_scan_kernel) take the representative's tables, root means and step counters, and every
// initial-state game takes the snapshot of its own act_iteration from the representative's history: what solving the copy
// would have left, bit for bit.  Only the template's (N - 1) x H entries are copied, as a solve writes only those.
template <typename real>
__global__ void __launch_bounds__(128) sp_share_kernel(SpDev p, CfrDev<real> d) {
  const int g = blockIdx.x;
  if (!p.sg_init[g]) return;
  const int rep = p.wave[3], E = (p.tmpl[0].N - 1) * p.H;
  const size_t st = p.table_stride;
  const real* __restrict__ hist = d.snap_hist + (size_t)d.sg_act_iter[g] * st;
  real* __restrict__ snap = d.Snap + (size_t)g * st;
  for (int i = threadIdx.x; i < E; i += blockDim.x) snap[i] = hist[i];
  if (g == rep) return;
  const size_t to = (size_t)g * st, from = (size_t)rep * st;
  const bool keep = d.keep_sum || d.fp;          // as cfr_launch_iter_d2 chooses its instantiation
  for (int i = threadIdx.x; i < E; i += blockDim.x) {
    d.R[to + i] = d.R[from + i];
    d.Sg[to + i] = d.Sg[from + i];
    if (keep) d.S[to + i] = d.S[from + i];
  }
  for (int i = threadIdx.x; i < 2 * p.H; i += blockDim.x) d.mu[(size_t)g * 2 * p.H + i] = d.mu[(size_t)rep * 2 * p.H + i];
  if (threadIdx.x < 2) d.steps[2 * g + threadIdx.x] = d.steps[2 * rep + threadIdx.x];
}

// update_value_network (subgame_solving.cc:672-676, add_training_example :220-226) of every finished subgame: for traverser
// t in {0, 1} the root query row (write_query_to :104-123; the root reach is the subgame's input beliefs) and float(mu[t]).
template <typename real>
__global__ void __launch_bounds__(128) sp_examples_kernel(SpDev p, const real* __restrict__ mu, float* __restrict__ ex_q,
                                                          float* __restrict__ ex_v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * p.K) return;
  const int g = i >> 1, t = i & 1;
  const int A = p.A, H = p.H, Q = p.Q;
  float* q = ex_q + (size_t)i * Q;
  q[0] = (float)p.g_player[g];
  q[1] = (float)t;
  const int lb = p.g_last_bid[g];
  for (int a = 0; a < A; ++a) q[2 + a] = (a == lb) ? 1.f : 0.f;
  const double* b = p.g_beliefs + (size_t)g * 2 * H;
  for (int pl = 0; pl < 2; ++pl) {
    double s = 0;
    for (int h = 0; h < H; ++h) s += b[pl * H + h] + 1e-80;
    for (int h = 0; h < H; ++h) q[2 + A + pl * H + h] = (float)((b[pl * H + h] + 1e-80) / s);
  }
  for (int h = 0; h < H; ++h) ex_v[(size_t)i * H + h] = (float)mu[((size_t)g * 2 + t) * H + h];
}

// sample_state (recursive_solving.cc:184-275) of every game with the snapshot of its subgame's sampling strategy taken at
// act_iteration, stored compactly as [edge = child - 1][hand].
template <typename real>
__global__ void __launch_bounds__(128) sp_advance_kernel(SpDev p, const real* __restrict__ snap) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.K) return;
  const int A = p.A, H = p.H;
  SpRng rng{p.mt + g, p.K, p.mt_idx[g]};
  int last_bid = p.g_last_bid[g], player = p.g_player[g];
  const TemplateDev t = p.tmpl[last_bid + 1];
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ nchild = p.nchild + t.node_off;
  const int* __restrict__ nbid = p.last_bid + t.node_off;
  const real* __restrict__ sigma = snap + (size_t)g * p.table_stride;
  double* bel = p.g_beliefs + (size_t)g * 2 * H;
  // policy[hand][action] of node n: dense over all actions in the reference, zero outside the legal range
  auto sig = [&](int n, int hand, int action) -> double {
    const int lo = nbid[n] < 0 ? 0 : nbid[n] + 1;
    const int j = action - lo;
    if (j < 0 || j >= nchild[n]) return 0.0;
    return (double)sigma[(size_t)(child_begin[n] + j - 1) * H + hand];
  };
  const int br_sampler = rng.uniform_int(0, 1);
  if (p.sample_leaf) {
    double sb[2 * kSpMaxH];
    for (int i = 0; i < 2 * H; ++i) sb[i] = bel[i];
    int path_n[kSpMaxPath], path_a[kSpMaxPath], plen = 0;
    int node = 0, depth = 0;
    while (nchild[node]) {
      const float eps = rng.canonical_f();
      const int pid = player ^ (depth & 1);
      const int lo = nbid[node] < 0 ? 0 : nbid[node] + 1, hi = nbid[node] < 0 ? A - 1 : A;   // get_bid_range, liars_dice.h:110-115
      int action;
      if (pid == br_sampler && eps < p.random_action_prob) {
        action = rng.uniform_int(lo, hi - 1);
      } else {
        const double* w = sb + pid * H;
        const int hand = sp_discrete(rng, H, [&](int i) { return w[i]; });
        action = sp_discrete(rng, A, [&](int a) { return sig(node, hand, a); });
      }
      for (int h = 0; h < H; ++h) sb[pid * H + h] *= sig(node, h, action);
      sp_normalize(sb + pid * H, H);
      if (plen < kSpMaxPath) { path_n[plen] = node; path_a[plen] = action; ++plen; }
      node = child_begin[node] + action - lo;
      ++depth;
    }
    for (int i = 0; i < plen; ++i) {     // second pass with the belief-propagation strategy (:232-245)
      const int n = path_n[i], action = path_a[i];
      const int lo = last_bid < 0 ? 0 : last_bid + 1;
      for (int h = 0; h < H; ++h) bel[player * H + h] *= sig(n, h, action);
      sp_normalize(bel + player * H, H);
      last_bid = nbid[child_begin[n] + action - lo];
      player ^= 1;
    }
  } else {
    const float eps = rng.canonical_f();
    const int lo = last_bid < 0 ? 0 : last_bid + 1, hi = last_bid < 0 ? A - 1 : A;
    int action;
    if (player == br_sampler && eps < p.random_action_prob) {
      action = rng.uniform_int(lo, hi - 1);
    } else {
      const double* w = bel + player * H;
      const int hand = sp_discrete(rng, H, [&](int i) { return w[i]; });
      action = sp_discrete(rng, A, [&](int a) { return sig(0, hand, a); });
    }
    for (int h = 0; h < H; ++h) bel[player * H + h] *= sig(0, h, action);
    sp_normalize(bel + player * H, H);
    last_bid = action;
    player ^= 1;
  }
  if (last_bid == A - 1) {               // terminal: RlRunner::step returns; the next call starts a new game (:161-163)
    last_bid = -1; player = 0;
    for (int i = 0; i < 2 * H; ++i) bel[i] = 1.0 / H;
  }
  p.g_last_bid[g] = last_bid; p.g_player[g] = player;
  p.mt_idx[g] = rng.idx;
}

}  // namespace cfrb
