// Parameter structs mirrored to Python by the `rela` module, field for field like the reference's
// liars_dice::SubgameSolvingParams (subgame_solving.h:43-58) and RecursiveSolvingParams (recursive_solving.h:31-38).
// cfvpy/selfplay.py fills them with setattr from cfg.env (selfplay.py:587-610) and raises on unknown keys, so the
// GPU-specific knobs below are ordinary extra fields with defaults: they can be set as `env.concurrent_games=...`
// without touching selfplay.py, and are invisible to configs that do not mention them.
#pragma once
#include <cstdlib>

#include "../../../include/cfrb200.h"

namespace liars_dice {

struct SubgameSolvingParams {
  int num_iters = 10;
  int max_depth = 2;
  bool linear_update = false;
  bool use_cfr = false;   // false = fictitious play (the YAML default), true = CFR; both run on the GPU
  bool optimistic = false;
  bool dcfr = false;
  double dcfr_alpha = 0;
  double dcfr_beta = 0;
  double dcfr_gamma = 0;
};

inline int env_int(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return v && *v ? std::atoi(v) : dflt;
}

struct RecursiveSolvingParams {
  int num_dice = 0;
  int num_faces = 0;
  float random_action_prob = 1.0f;
  bool sample_leaf = false;
  SubgameSolvingParams subgame_params;
  // ---- rebel_b200 extensions
  int concurrent_games = env_int("CFRB_CONCURRENT_GAMES", 1024);   // self-play games advanced in lock-step per thread loop
  int net_mode = env_int("CFRB_NET_MODE", 3);                      // include/cfrb200.h CFRB_NET_*: 3 = wgmma fp16 operands, fast tanh GELU
  int state_dtype = env_int("CFRB_STATE_DTYPE", 0);                // CFRB_STATE_*: 0 = fp64 tables
  int host_walk = env_int("CFRB_HOST_WALK", 0);                    // 1 = per-game sampling on the host (parity mode of the device walk)
};

// A tensor-core net mode falls back to the fp32 SIMT net only on games whose Net2 weights do not fit a tensor-core kernel
// (cfrb_tc_net_supported: 2x7f, 3x4f, 6x2f, 2x8f, one-die games from 1x33f on, ...).
inline int effective_net_mode(const RecursiveSolvingParams& p) {
  return (p.net_mode >= 2 && !cfrb_tc_net_supported(p.num_dice, p.num_faces, 256)) ? 1 : p.net_mode;
}

// The handle configuration of a recursive solver with these parameters and `capacity` subgames per wave.
inline cfrb_config solver_config(const RecursiveSolvingParams& cfg, int device, int capacity) {
  const auto& sp = cfg.subgame_params;
  cfrb_config c{};
  c.solver = sp.use_cfr ? CFRB_SOLVER_CFR : CFRB_SOLVER_FP;
  c.optimistic = sp.optimistic;
  c.num_dice = cfg.num_dice; c.num_faces = cfg.num_faces; c.max_depth = sp.max_depth; c.num_iters = sp.num_iters;
  c.linear_update = sp.linear_update; c.dcfr = sp.dcfr; c.dcfr_alpha = sp.dcfr_alpha; c.dcfr_beta = sp.dcfr_beta;
  c.dcfr_gamma = sp.dcfr_gamma; c.max_subgames = capacity; c.device = device; c.net_mode = effective_net_mode(cfg); c.hidden = 256;
  c.state_dtype = cfg.state_dtype;
  return c;
}

}  // namespace liars_dice
