"""TEST INFRASTRUCTURE — ctypes front-end for the CPU oracle.

Two back-ends with the same call surface:

* ``Oracle("port")``       -> oracle/libcfr_oracle.so, the plain-C restatement (cfr_oracle.c);
* ``Oracle("ref_nofma")`` / ``Oracle("ref_fast")`` -> oracle/_ref/libref_*.so, the reference's own
  C++ sources compiled where they lie (oracle/Makefile, ref_harness.cc).

Only tests/, ``__graft_entry__.smoke()`` and bench.py's ``cpu_baseline`` / ``--impl reference``
legs may import this module.  rebel_b200/ never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {
    "port": ("libcfr_oracle.so", "orc_"),
    "ref_nofma": (os.path.join("_ref", "libref_nofma.so"), "ref_"),
    "ref_fast": (os.path.join("_ref", "libref_fast.so"), "ref_"),
}

_dp = C.POINTER(C.c_double)
_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)


def _ptr(a, t):
    return None if a is None else a.ctypes.data_as(t)


def build_port():
    subprocess.check_call(["make", "-s", "-C", _HERE, "libcfr_oracle.so"])


def build_ref():
    """Only possible where a checkout of the original project exists (REBEL_REFERENCE, default in oracle/Makefile)."""
    subprocess.check_call(["make", "-s", "-j8", "-C", _HERE, "ref"])


def available(kind):
    return os.path.exists(os.path.join(_HERE, _LIBS[kind][0]))


def game_dims(D, F):
    A = 1 + 2 * D * F
    H = F ** D
    return A, H, 2 + A + 2 * H


class Oracle:
    def __init__(self, kind="port"):
        rel, self.pfx = _LIBS[kind]
        path = os.path.join(_HERE, rel)
        if kind == "port" and not os.path.exists(path):
            build_port()
        if kind != "port":
            import torch  # noqa: F401  (libref links libtorch; make sure its libs are loaded)
        self.kind = kind
        self.lib = C.CDLL(path)
        f = self._f("bench_solve")
        f.restype = C.c_double
        if kind != "port":
            self._f("bench_datagen").restype = C.c_int64
            self._f("bench_datagen_windows").restype = C.c_int64
            self._f("last_error").restype = C.c_char_p

    def _f(self, name):
        return getattr(self.lib, self.pfx + name)

    # -- integers ---------------------------------------------------------------------------
    def unroll_tree(self, D, F, last_bid=-1, player_id=0, max_depth=1000000):
        cap = 1 << 16
        out = np.zeros((cap, 6), np.int32)
        n = self._f("unroll_tree")(int(D), int(F), int(last_bid), int(player_id), int(max_depth), _ptr(out, _ip), cap)
        assert n > 0, n
        return out[:n].copy()

    def num_matches(self, D, F, hand, face):
        return self._f("num_matches")(int(D), int(F), int(hand), int(face))

    # -- small fp ---------------------------------------------------------------------------
    def win_probability(self, D, F, bet, beliefs):
        b = np.ascontiguousarray(beliefs, np.float64)
        out = np.zeros(F ** D, np.float64)
        self._f("win_probability")(int(D), int(F), int(bet), _ptr(b, _dp), _ptr(out, _dp))
        return out

    def query(self, D, F, traverser, last_bid, player_id, r0, r1):
        A, H, Q = game_dims(D, F)
        r0 = np.ascontiguousarray(r0, np.float64)
        r1 = np.ascontiguousarray(r1, np.float64)
        out = np.zeros(Q, np.float32)
        n = self._f("query")(int(D), int(F), int(traverser), int(last_bid), int(player_id), _ptr(r0, _dp), _ptr(r1, _dp),
                             _ptr(out, _fp))
        assert n == Q
        return out

    def synthetic_beliefs(self, H, seed):
        out = np.zeros((2, H), np.float64)
        self._f("synthetic_beliefs")(int(H), int(seed), _ptr(out, _dp))
        return out

    # -- CFR --------------------------------------------------------------------------------
    def cfr_solve(self, D, F, beliefs, checkpoints, last_bid=-1, player_id=0, num_iters=1024, max_depth=2,
                  linear_update=True, dcfr=False, dcfr_alpha=0.0, dcfr_beta=0.0, dcfr_gamma=0.0,
                  net_w=None, hidden=256, want=("regrets", "last", "sum", "avg", "root_means")):
        """Returns dict of arrays indexed [checkpoint, ...]; dense tables are [C,N,H,A] fp64."""
        A, H, Q = game_dims(D, F)
        tree = self.unroll_tree(D, F, last_bid, player_id, max_depth)
        N = len(tree)
        nchild = tree[:, 3] - tree[:, 2]
        L = int(((nchild == 0) & (tree[:, 0] != A - 1)).sum())
        cps = np.ascontiguousarray(checkpoints, np.int32)
        Cn = len(cps)
        b = np.ascontiguousarray(beliefs, np.float64).reshape(2, H)
        w = None if net_w is None else np.ascontiguousarray(net_w, np.float32)
        bufs = {k: np.zeros((Cn, N, H, A), np.float64) for k in ("regrets", "last", "sum", "avg") if k in want}
        rm = np.zeros((Cn, 2, H), np.float64)
        lv = np.zeros((Cn, max(L, 1), H), np.float32)
        qs = np.zeros((Cn, max(L, 1), Q), np.float32)
        tv = np.zeros((Cn, N, H), np.float64)
        f = self._f("cfr_solve")
        f.argtypes = [C.c_int] * 4 + [_dp] + [C.c_int] * 4 + [C.c_double] * 3 + [_fp, C.c_int, C.c_int, _ip] + \
            [_dp] * 5 + [_fp, _fp, _dp]
        n = f(int(D), int(F), int(last_bid), int(player_id), _ptr(b, _dp), int(num_iters), int(max_depth), int(linear_update), int(dcfr),
              dcfr_alpha, dcfr_beta, dcfr_gamma, _ptr(w, _fp), hidden, Cn, _ptr(cps, _ip),
              _ptr(bufs.get("regrets"), _dp), _ptr(bufs.get("last"), _dp), _ptr(bufs.get("sum"), _dp),
              _ptr(bufs.get("avg"), _dp), _ptr(rm, _dp), _ptr(lv, _fp), _ptr(qs, _fp), _ptr(tv, _dp))
        assert n == N, (n, N)
        out = dict(bufs)
        out.update(root_means=rm, leaf_values=lv[:, :L], queries=qs[:, :L], traverser_values=tv, tree=tree,
                   pleaf=np.nonzero((nchild == 0) & (tree[:, 0] != A - 1))[0],
                   term=np.nonzero(tree[:, 0] == A - 1)[0])
        return out

    def fp_solve(self, D, F, beliefs, checkpoints, last_bid=-1, player_id=0, num_iters=1024, max_depth=2, linear_update=True,
                 optimistic=False, net_w=None, hidden=256):
        """Fictitious play (FP, subgame_solving.cc:364-506): dict of [C,N,H,A] tables last / sum / avg and root_means."""
        A, H, Q = game_dims(D, F)
        N = len(self.unroll_tree(D, F, last_bid, player_id, max_depth))
        cps = np.ascontiguousarray(checkpoints, np.int32)
        b = np.ascontiguousarray(beliefs, np.float64).reshape(2, H)
        w = None if net_w is None else np.ascontiguousarray(net_w, np.float32)
        bufs = {k: np.zeros((len(cps), N, H, A), np.float64) for k in ("last", "sum", "avg")}
        rm = np.zeros((len(cps), 2, H), np.float64)
        f = self._f("fp_solve")
        f.argtypes = [C.c_int] * 4 + [_dp] + [C.c_int] * 4 + [_fp, C.c_int, C.c_int, _ip] + [_dp] * 4
        n = f(int(D), int(F), int(last_bid), int(player_id), _ptr(b, _dp), int(num_iters), int(max_depth), int(linear_update),
              int(optimistic), _ptr(w, _fp), hidden, len(cps), _ptr(cps, _ip), _ptr(bufs["last"], _dp), _ptr(bufs["sum"], _dp),
              _ptr(bufs["avg"], _dp), _ptr(rm, _dp))
        assert n == N, (n, N)
        out = dict(bufs)
        out["root_means"] = rm
        return out

    def net_evaluation(self, D, F, net_w, num_iters=64, max_depth=2, linear_update=True, use_cfr=True, hidden=256, what=3):
        """rela/pybind.cc:45-84 with flat Net2 weights: dict with strategy_recursive / strategy_to_leaf
        [N,H,A] and values = [expl(recursive), expl(to_leaf), eval_net mse (net beliefs), eval_net mse (full-tree beliefs)]."""
        A, H, Q = game_dims(D, F)
        N = len(self.unroll_tree(D, F))
        sr, sl = np.zeros((N, H, A)), np.zeros((N, H, A))
        out = np.zeros(4)
        w = np.ascontiguousarray(net_w, np.float32)
        f = self._f("net_evaluation")
        f.argtypes = [C.c_int] * 6 + [_fp] + [C.c_int] * 2 + [_dp] * 3
        n = f(int(D), int(F), int(num_iters), int(max_depth), int(linear_update), int(use_cfr), _ptr(w, _fp), hidden, int(what),
              _ptr(sr, _dp), _ptr(sl, _dp), _ptr(out, _dp))
        if n < 0:
            raise RuntimeError(self._f("last_error")().decode())
        return {"strategy_recursive": sr, "strategy_to_leaf": sl, "values": out}

    def exploitability(self, D, F, strategy):
        s = np.ascontiguousarray(strategy, np.float64)
        out = np.zeros(2, np.float64)
        rc = self._f("exploitability")(D, F, _ptr(s, _dp), _ptr(out, _dp))
        assert rc == 0
        return out

    def set_net_noise(self, rel, seed=0):
        """Reference builds only: relative gaussian noise on the Net2 outputs of the following cfr_solve calls (this thread)."""
        assert self.kind != "port"
        f = self.lib.ref_set_net_noise
        f.argtypes = [C.c_double, C.c_uint64]
        f.restype = None
        f(float(rel), int(seed))

    def set_net_emulation(self, model):
        """Reference builds only: 0 = the reference's fp32 ATen net, 1 / 2 = arithmetic model of the tensor-core value-net kernels
        (fp16 operands; fp32 GELU / packed-half GELU) inside the reference's net, for cfr_solve and rl_runner on this thread."""
        assert self.kind != "port"
        f = self.lib.ref_set_net_emulation
        f.argtypes = [C.c_int]
        f.restype = None
        f(int(model))

    def rl_runner(self, D, F, seed, n_games, num_iters=1024, max_depth=2, linear_update=True,
                  random_action_prob=0.25, sample_leaf=True, net_w=None, hidden=256, cap=4096, use_cfr=True, optimistic=False,
                  dcfr=False, dcfr_alpha=0.0, dcfr_beta=0.0, dcfr_gamma=0.0, max_subgames=0, trace=False):
        """RlRunner::step n_games times (recursive_solving.cc:160-182): the training examples (q [n, Q], v [n, H]), two per solved
        subgame.  use_cfr=False is fictitious play (optimistic applies), use_cfr with dcfr is DCFR(alpha, beta, gamma).
        Port only: max_subgames > 0 stops after that many subgames, and trace=True also returns one int32 row per subgame:
        (game index, root last_bid, root player, act_iteration, br_sampler)."""
        A, H, Q = game_dims(D, F)
        q = np.zeros((cap, Q), np.float32)
        v = np.zeros((cap, H), np.float32)
        tr = np.zeros((cap // 2 + 1, 5), np.int32) if trace else None
        w = None if net_w is None else np.ascontiguousarray(net_w, np.float32)
        f = self._f("rl_runner")
        f.argtypes = [C.c_int] * 5 + [C.c_float] + [C.c_int] * 3 + [_fp, C.c_int, _fp, _fp] + [C.c_int] * 4 + [C.c_double] * 3 + \
            [C.c_int, _ip, C.c_int]
        n = f(D, F, num_iters, max_depth, int(linear_update), random_action_prob, int(sample_leaf), seed, n_games,
              _ptr(w, _fp), hidden, _ptr(q, _fp), _ptr(v, _fp), cap, int(use_cfr), int(optimistic), int(dcfr), float(dcfr_alpha),
              float(dcfr_beta), float(dcfr_gamma), int(max_subgames), _ptr(tr, _ip), 0 if tr is None else len(tr))
        if n < 0:
            raise RuntimeError(self._f("last_error")().decode())
        assert n <= cap, (n, cap)
        if trace:
            return q[:n].copy(), v[:n].copy(), tr[:n // 2].copy()
        return q[:n].copy(), v[:n].copy()

    def sampled_strategy(self, D, F, seed, num_iters=1024, max_depth=2, linear_update=True, net_w=None, hidden=256):
        """compute_sampled_strategy_recursive_to_leaf: dense [N_full, H, A]."""
        A, H, Q = game_dims(D, F)
        N = len(self.unroll_tree(D, F))
        out = np.zeros((N, H, A), np.float64)
        w = None if net_w is None else np.ascontiguousarray(net_w, np.float32)
        f = self._f("sampled_strategy")
        f.argtypes = [C.c_int] * 6 + [_fp, C.c_int, _dp]
        n = f(D, F, num_iters, max_depth, int(linear_update), seed, _ptr(w, _fp), hidden, _ptr(out, _dp))
        if n < 0:
            raise RuntimeError(self._f("last_error")().decode())
        assert n == N
        return out

    def strategy_reach(self, D, F, strategy):
        A, H, Q = game_dims(D, F)
        s = np.ascontiguousarray(strategy, np.float64)
        out = np.zeros((2, s.shape[0], H), np.float64)
        n = self._f("strategy_reach")(int(D), int(F), _ptr(s, _dp), _ptr(out, _dp))
        assert n == s.shape[0]
        return out

    def net2_forward(self, w, Q, hidden, H, queries):
        assert self.kind == "port"
        w = np.ascontiguousarray(w, np.float32)
        x = np.ascontiguousarray(queries, np.float32)
        out = np.zeros((x.shape[0], H), np.float32)
        self.lib.orc_net2_forward(_ptr(w, _fp), Q, hidden, H, _ptr(x, _fp), x.shape[0], _ptr(out, _fp))
        return out

    # -- timed baselines --------------------------------------------------------------------
    def bench_solve(self, D, F, n_subgames, seed0=0, last_bid=-1, player_id=0, num_iters=1024, max_depth=2,
                    net_w=None, hidden=256, script_path=None, threads=1, want_means=False, beliefs=None):
        """Seconds to solve n root subgames with synthetic beliefs.  port: single thread, C Net2 from flat
        weights.  ref_*: `threads` std::threads, TorchScript Net2 from script_path (zero net if None)."""
        A, H, Q = game_dims(D, F)
        rm = np.zeros((n_subgames, 2, H), np.float64) if want_means else None
        bl = None
        if beliefs is not None:
            bl = np.ascontiguousarray(beliefs, np.float64)
            assert bl.shape == (n_subgames, 2, H)
        f = self._f("bench_solve")
        if self.kind == "port":
            w = None if net_w is None else np.ascontiguousarray(net_w, np.float32)
            f.argtypes = [C.c_int] * 8 + [_fp, C.c_int, _dp, _dp]
            secs = f(D, F, last_bid, player_id, num_iters, max_depth, n_subgames, seed0, _ptr(w, _fp), hidden,
                     _ptr(rm, _dp), _ptr(bl, _dp))
        else:
            f.argtypes = [C.c_int] * 8 + [C.c_char_p, C.c_int, _dp, _dp]
            secs = f(D, F, last_bid, player_id, num_iters, max_depth, n_subgames, seed0,
                     (script_path or "").encode(), threads, _ptr(rm, _dp), _ptr(bl, _dp))
            if secs < 0:
                raise RuntimeError(self._f("last_error")().decode())
        return (secs, rm) if want_means else secs

    def bench_datagen(self, D, F, script_path, threads, seconds, seed0=0, num_iters=1024, max_depth=2,
                      random_action_prob=0.25, sample_leaf=True):
        assert self.kind != "port"
        el = C.c_double(0)
        f = self._f("bench_datagen")
        f.argtypes = [C.c_int] * 4 + [C.c_float, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_double, _dp]
        n = f(D, F, num_iters, max_depth, random_action_prob, int(sample_leaf), script_path.encode(), threads, seed0,
              float(seconds), C.byref(el))
        if n < 0:
            raise RuntimeError(self._f("last_error")().decode())
        return n, el.value

    def bench_datagen_windows(self, D, F, script_path, threads, warmup_s, n_windows, window_s, seed0=0, num_iters=1024, max_depth=2,
                              random_action_prob=0.25, sample_leaf=True):
        """One continuous run of `threads` RlRunner loops; returns (examples per window [n], seconds per window [n])."""
        assert self.kind != "port"
        counts = np.zeros(n_windows, np.int64)
        secs = np.zeros(n_windows, np.float64)
        f = self._f("bench_datagen_windows")
        f.argtypes = [C.c_int] * 4 + [C.c_float, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double,
                      C.POINTER(C.c_int64), _dp]
        n = f(D, F, num_iters, max_depth, random_action_prob, int(sample_leaf), script_path.encode(), threads, seed0,
              float(warmup_s), n_windows, float(window_s), counts.ctypes.data_as(C.POINTER(C.c_int64)), _ptr(secs, _dp))
        if n < 0:
            raise RuntimeError(self._f("last_error")().decode())
        return counts, secs
