"""Plays one seeded run of every kind of match, LBR and agent that libcfrb200 builds, and saves everything each one returns, so
that two builds of the library can be compared bit for bit.  1x4f, depth 2, CFR with the seed-0 fp32 Net2:

  create average and sampled; create2 every-node vs average and sampled vs every-node; create3 blueprint vs a sampled handle and
  blueprint vs blueprint; create_lbr, create_lbr2 every-node and create_lbr_blueprint; a scripted game sequence through
  cfrb_agent_create (sampled) and cfrb_agent_create_blueprint.

Saved per run: payoffs, plies, solves, subgame iterations, per-agent solves, the traces of games 0 and 1, the handles' kernel
launch counts; for LBR its traces and counts; for the agents every action played, its probability rows and the agent's counts.
The blueprint is the full-game CFR solve of 1x4f after 64 iterations.

    python scripts/match_kinds_check.py --lib path/to/libcfrb200.so --out a.npz
    python scripts/match_kinds_check.py --compare a.npz b.npz"""
import argparse
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

D, F, SLOTS, GAMES, ITERS, SEED = 1, 4, 32, 64, 64, 5


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        x, y = a[k], b[k]
        bits = [np.frombuffer(v.tobytes(), np.uint8) for v in (x, y)]   # bit for bit: NaNs and signed zeros included
        if x.dtype != y.dtype or x.shape != y.shape or not np.array_equal(*bits):
            bad.append(k)
    print(f"{len(a.files)} arrays in {a_path}, {len(b.files)} in {b_path}: " + ("all bit-identical" if not bad else f"differ: {bad}"))
    return 0 if not bad else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", type=str, help="the libcfrb200.so to load")
    ap.add_argument("--out", type=str, default="match_kinds.npz")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        return compare(*args.compare)
    from rebel_b200 import capi
    if args.lib:
        capi.LIB_PATH = os.path.abspath(args.lib)
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    L = capi.lib()
    vp = C.c_void_p
    L.cfrb_agent_create.argtypes = [vp, C.c_int32, C.c_uint64, C.c_int32, C.POINTER(vp)]
    L.cfrb_agent_create_blueprint.argtypes = [vp, C.c_int32, C.c_uint64, C.POINTER(vp)]
    L.cfrb_agent_new_games.argtypes = [vp, C.c_int32, vp, vp, vp, vp]
    L.cfrb_agent_step.argtypes = [vp, C.c_int32, vp, vp, vp, vp]
    L.cfrb_agent_counts.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.cfrb_agent_destroy.argtypes = [vp]

    w = flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict())
    hs = []
    for _ in range(2):
        S = capi.WaveSolver(D, F, SLOTS, max_depth=2, num_iters=ITERS, linear_update=True, net_mode=capi.NET_FP32,
                            solver=capi.SOLVER_CFR)
        S.set_weights(w)
        S.sync()
        hs.append(S)
    a, b = hs
    fg = capi.FullGame(D, F)
    fg.step(64)
    bp = capi.Blueprint.from_full_game(fg)
    fg.close()
    out = {}

    def record(name, M, lbr=False):
        r = M.play()
        for k, v in r.items():
            out[f"{name}/{k}"] = np.asarray(v)
        for g in (0, 1):
            for k, v in M.trace(g).items():
                out[f"{name}/trace{g}/{k}"] = v
            if lbr:
                for k, v in M.lbr_trace(g).items():
                    out[f"{name}/lbr_trace{g}/{k}"] = v
        out[f"{name}/launches"] = np.array([a.kernel_launches, b.kernel_launches], np.int64)
        M.close()

    A_, S_, E_ = capi.MATCH_AVERAGE, capi.MATCH_SAMPLED, capi.MATCH_EVERY_NODE
    record("create_average", capi.Match(a, b, SLOTS, GAMES, seed=SEED, policy=A_))
    record("create_sampled", capi.Match(a, b, SLOTS, GAMES, seed=SEED, policy=S_))
    record("create2_every_node_vs_average", capi.Match(a, b, SLOTS, GAMES, seed=SEED, policy=E_, policy_b=A_))
    record("create2_sampled_vs_every_node", capi.Match(a, b, SLOTS, GAMES, seed=SEED, policy=S_, policy_b=E_))
    record("create3_blueprint_vs_sampled", capi.Match(bp, b, SLOTS, GAMES, seed=SEED, policy=S_))
    record("create3_blueprint_vs_blueprint", capi.Match(bp, bp, SLOTS, GAMES, seed=SEED))
    record("create_lbr", capi.LbrMatch(a, SLOTS, GAMES, seed=SEED), lbr=True)
    record("create_lbr2_every_node", capi.LbrMatch(a, SLOTS, GAMES, seed=SEED, policy=E_), lbr=True)
    record("create_lbr_blueprint", capi.LbrMatch(bp, SLOTS, GAMES, seed=SEED), lbr=True)

    def agent_games(name, create):
        """Games on 8 tables to their ends, one step call per round, against a seeded uniform-random legal opponent."""
        ag = vp()
        capi._check(create(C.byref(ag)))
        A, H, n = 2 * D * F + 1, F ** D, 8
        rng = np.random.RandomState(SEED)
        ids = np.arange(n, dtype=np.int32)
        seats = (ids % 2).astype(np.int32)
        hands = rng.randint(0, H, size=n).astype(np.int32)
        keys = np.arange(n, dtype=np.uint64)
        capi._check(L.cfrb_agent_new_games(ag, n, ids.ctypes.data, seats.ctypes.data, hands.ctypes.data, keys.ctypes.data))
        lb, player, running = np.full(n, -1), np.zeros(n, np.int64), np.ones(n, bool)
        acts_log, probs_log = [], []
        while running.any():
            live = np.flatnonzero(running).astype(np.int32)
            lo = np.where(lb[live] < 0, 0, lb[live] + 1)
            hi = np.where(lb[live] < 0, A - 1, A)
            mine = player[live] == seats[live]
            acts = np.where(mine, -1, lo + (rng.rand(len(live)) * (hi - lo)).astype(np.int64)).astype(np.int32)
            probs = np.zeros((len(live), A), np.float64)
            done = np.zeros(len(live), np.int32)
            capi._check(L.cfrb_agent_step(ag, len(live), live.ctypes.data, acts.ctypes.data, probs.ctypes.data, done.ctypes.data))
            acts_log.append(np.stack([live, acts]))
            probs_log.append(probs)
            lb[live] = acts
            player[live] ^= 1
            running[live[done == 1]] = False
        solves, iters = C.c_int64(0), C.c_int64(0)
        capi._check(L.cfrb_agent_counts(ag, C.byref(solves), C.byref(iters)))
        L.cfrb_agent_destroy(ag)
        out[f"{name}/actions"] = np.concatenate(acts_log, axis=1)
        out[f"{name}/probs"] = np.concatenate(probs_log)
        out[f"{name}/counts"] = np.array([solves.value, iters.value, a.kernel_launches], np.int64)

    agent_games("agent_sampled", lambda o: L.cfrb_agent_create(a._h, 8, SEED, S_, o))
    agent_games("agent_blueprint", lambda o: L.cfrb_agent_create_blueprint(bp._b, 8, SEED, o))
    bp.close()
    a.close()
    b.close()
    np.savez(args.out, **out)
    print(f"{len(out)} arrays from {capi.LIB_PATH} to {args.out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
