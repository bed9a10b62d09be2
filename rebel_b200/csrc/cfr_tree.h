// Host-side Liar's Dice public-tree templates for the CFR wave solver.
//
// The reference rebuilds `vector<UnrolledTreeNode>` for every subgame (subgame_solving.cc:530 ->
// tree.h:51-70).  The shape of a depth-limited subgame tree depends only on (root last_bid, max_depth),
// and the acting player of a node is root_player XOR (depth & 1), so here every distinct root bid gets
// ONE immutable template, built once per handle and shared by all subgames of all waves.
//
// Indexing contract (bit-exact with the reference, pinned by tests against tree_test.cc:20-125):
//   * nodes are in the reference's BFS order; children of node n are [child_begin, child_begin+nchild)
//     and child j corresponds to action act_lo + j (tree.h:81-107);
//   * every non-root node c has exactly one incoming edge, so per-(node,hand,action) tables
//     [n][h][a] are stored compactly as [edge = c-1][h] with c = child(n, a).
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace cfrb {

struct GameShape {
  int D = 0, F = 0, A = 0, H = 0, Q = 0, liar = 0;
  GameShape() = default;
  GameShape(int d, int f) : D(d), F(f) {
    A = 1 + 2 * d * f;                 // liars_dice.h:55
    H = 1;
    for (int i = 0; i < d; ++i) H *= f;  // liars_dice.h:56
    liar = A - 1;                      // liars_dice.h:57
    Q = 2 + A + 2 * H;                 // subgame_solving.cc:100-102
  }
  // liars_dice.h:110-115
  void bid_range(int last_bid, int* lo, int* hi) const {
    if (last_bid < 0) { *lo = 0; *hi = A - 1; } else { *lo = last_bid + 1; *hi = A; }
  }
  // liars_dice.h:83-91 (last face is wild)
  int num_matches(int hand, int face) const {
    int m = 0;
    for (int i = 0; i < D; ++i) { int d = hand % F; m += (d == face || d == F - 1); hand /= F; }
    return m;
  }
};

enum NodeKind : int32_t { kInner = 0, kTerminal = 1, kPseudoLeaf = 2 };

// One template = one unrolled tree for root bid `root_bid` (player parity factored out).
struct TreeTemplate {
  int root_bid = -1;
  int N = 0, L = 0, T = 0, levels = 0;   // nodes, pseudo-leaves, terminals, depth levels (max depth + 1)
  std::vector<int32_t> parent, child_begin, nchild, last_bid, depth, kind, slot, act_lo;
  std::vector<int32_t> level_begin;       // [levels + 1]
  std::vector<int32_t> pleaf_node;        // [L] node ids, increasing
  std::vector<int32_t> term_node;         // [T]
};

inline TreeTemplate build_template(const GameShape& g, int root_bid, int max_depth) {
  TreeTemplate t;
  t.root_bid = root_bid;
  auto push = [&](int bid, int par, int dep) {
    t.last_bid.push_back(bid); t.parent.push_back(par); t.depth.push_back(dep);
    t.child_begin.push_back(0); t.nchild.push_back(0);
  };
  push(root_bid, -1, 0);
  for (size_t n = 0; n < t.last_bid.size() && t.depth[n] < max_depth; ++n) {
    int lo, hi;
    g.bid_range(t.last_bid[n], &lo, &hi);
    t.child_begin[n] = (int32_t)t.last_bid.size();
    t.nchild[n] = hi - lo;
    for (int a = lo; a < hi; ++a) push(a, (int)n, t.depth[n] + 1);
  }
  t.N = (int)t.last_bid.size();
  t.kind.assign(t.N, kInner); t.slot.assign(t.N, -1); t.act_lo.assign(t.N, 0);
  for (int n = 0; n < t.N; ++n) {
    int lo, hi;
    g.bid_range(t.last_bid[n], &lo, &hi);
    t.act_lo[n] = lo;
    if (t.last_bid[n] == g.liar) { t.kind[n] = kTerminal; t.slot[n] = t.T++; t.term_node.push_back(n); }
    else if (t.nchild[n] == 0) { t.kind[n] = kPseudoLeaf; t.slot[n] = t.L++; t.pleaf_node.push_back(n); }
  }
  t.levels = t.depth[t.N - 1] + 1;   // BFS order: last node is deepest
  t.level_begin.assign(t.levels + 1, t.N);
  for (int n = t.N - 1; n >= 0; --n) t.level_begin[t.depth[n]] = n;
  return t;
}

// Schedule of the depth <= 2 CFR kernel: a subgame's cost is its table items ((N - 1) edges x H hands) plus its value-net query
// rows (L).  The cost is not monotone in the root bid for every game, so templates are ranked by it: rank 0 = the costliest,
// ties by template index.
inline int64_t schedule_cost(const TreeTemplate& t, int H) { return (int64_t)(t.N - 1) * H + t.L; }
inline std::vector<int> schedule_ranks(const std::vector<TreeTemplate>& tmpl, int H) {
  std::vector<int> by_cost(tmpl.size()), rank(tmpl.size());
  for (size_t i = 0; i < tmpl.size(); ++i) by_cost[i] = (int)i;
  std::stable_sort(by_cost.begin(), by_cost.end(),
                   [&](int a, int b) { return schedule_cost(tmpl[a], H) > schedule_cost(tmpl[b], H); });
  for (size_t r = 0; r < by_cost.size(); ++r) rank[by_cost[r]] = (int)r;
  return rank;
}
// order[0..n) = the wave positions 0..n-1 of subgames with templates tm[], sorted by rank (stable counting sort); the same
// permutation sp_scan_kernel builds on the device
inline void schedule_order(const std::vector<int>& rank, const int* tm, int n, int* order) {
  std::vector<int> start(rank.size() + 1, 0);
  for (int k = 0; k < n; ++k) ++start[rank[tm[k]] + 1];
  for (size_t r = 1; r < start.size(); ++r) start[r] += start[r - 1];
  for (int k = 0; k < n; ++k) order[start[rank[tm[k]]]++] = k;
}

}  // namespace cfrb
