"""TEST INFRASTRUCTURE — ctypes front-end for the evaluation oracles of recursive_eval's report (compute_ev2,
compute_immediate_regrets, the fictitious-play sampled recursive strategy).

* ``EvRegretOracle("port")`` -> oracle/libev_regret_oracle.so, the plain-C restatement (ev_regret_oracle.c), built on first use;
* ``EvRegretOracle("ref")``  -> oracle/_ref/libref_eval_nofma.so, extern "C" wrappers (ref_eval_harness.cc) around the
  reference's own functions, linked with oracle/_ref/libref_nofma.so.  Only where a checkout of the original project exists
  (REBEL_REFERENCE, else the default location of oracle/Makefile); used to generate tests/golden/ev_regrets.npz.

Only tests/ and the fixture generators import this module.  rebel_b200/ never does.
"""
import ctypes as C
import os
import subprocess
import sys
import sysconfig

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PORT_LIB = os.path.join(_HERE, "libev_regret_oracle.so")
REF_LIB = os.path.join(_HERE, "_ref", "libref_eval_nofma.so")
DEFAULT_REFERENCE = "/root/reference"     # same default as oracle/Makefile

_dp = C.POINTER(C.c_double)


def game_dims(D, F):
    A = 1 + 2 * D * F
    H = F ** D
    return A, H, 2 + A + 2 * H


def _ptr(a):
    return a.ctypes.data_as(_dp)


def build_port():
    """gcc with the flags of the C oracle (oracle/Makefile): -O2 -ffp-contract=off, no fused multiply-adds."""
    subprocess.check_call(["gcc", "-std=gnu11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-o", PORT_LIB,
                           os.path.join(_HERE, "ev_regret_oracle.c"), "-lm"])


def build_ref():
    """The wrappers compiled against a checkout's headers with the deterministic flags of oracle/Makefile (-O2
    -ffp-contract=off) and linked with the reference library that `make -C oracle ref` builds."""
    import torch
    import pybind11
    ref = os.environ.get("REBEL_REFERENCE") or DEFAULT_REFERENCE
    src = os.path.join(ref, "csrc", "liars_dice")
    tdir = os.path.dirname(torch.__file__)
    if not os.path.exists(os.path.join(_HERE, "_ref", "libref_nofma.so")):
        subprocess.check_call(["make", "-s", "-j8", "-C", _HERE, "ref", "REF=" + os.path.abspath(ref)])
    subprocess.check_call(["g++", "-std=c++17", "-fPIC", "-shared", "-w", "-O2", "-ffp-contract=off",
                           "-include", "fstream", "-include", "iostream", "-include", "iomanip", "-include", "queue",
                           "-I" + src, "-I" + os.path.join(tdir, "include"), "-I" + os.path.join(tdir, "include", "torch", "csrc", "api", "include"),
                           "-I" + sysconfig.get_paths()["include"], "-I" + pybind11.get_include(),
                           "-o", REF_LIB, os.path.join(_HERE, "ref_eval_harness.cc"),
                           "-L" + os.path.join(_HERE, "_ref"), "-lref_nofma", "-Wl,-rpath,$ORIGIN",
                           "-L" + os.path.join(tdir, "lib"), "-ltorch", "-ltorch_cpu", "-lc10", "-Wl,-rpath," + os.path.join(tdir, "lib")])


class EvRegretOracle:
    def __init__(self, kind="port"):
        assert kind in ("port", "ref")
        self.kind = kind
        if kind == "port":
            if not os.path.exists(PORT_LIB):
                build_port()
            self.lib = C.CDLL(PORT_LIB)
            self.pfx = "evo_"
        else:
            import torch  # noqa: F401  (the reference library links libtorch)
            if not os.path.exists(REF_LIB):
                build_ref()
            self.lib = C.CDLL(REF_LIB)
            self.pfx = "refev_"
            self.lib.refev_last_error.restype = C.c_char_p

    def _f(self, name):
        return getattr(self.lib, self.pfx + name)

    def _check(self, rc):
        if rc < 0:
            raise RuntimeError(self.lib.refev_last_error().decode() if self.kind == "ref" else f"error {rc}")
        return rc

    def ev2(self, D, F, s1, s2):
        """compute_ev2 (subgame_solving.cc:975-982) of two dense full-tree strategies: [ev0, ev1]."""
        a = np.ascontiguousarray(s1, np.float64)
        b = np.ascontiguousarray(s2, np.float64)
        out = np.zeros(2, np.float64)
        f = self._f("ev2")
        f.argtypes = [C.c_int, C.c_int, _dp, _dp, _dp]
        self._check(f(int(D), int(F), _ptr(a), _ptr(b), _ptr(out)))
        return out

    def immediate_regrets(self, D, F, strategies):
        """compute_immediate_regrets (subgame_solving.cc:984-1050) of dense strategies [S, N, H, A]: [N, H]."""
        A, H, Q = game_dims(D, F)
        s = np.ascontiguousarray(strategies, np.float64)
        N = s.shape[1]
        out = np.zeros((N, H), np.float64)
        f = self._f("immediate_regrets")
        if self.kind == "port":
            sums = np.zeros((N, H, A), np.float64)
            f.argtypes = [C.c_int, C.c_int, _dp, C.c_int, _dp, C.c_int, _dp]
            n = f(int(D), int(F), _ptr(s), s.shape[0], _ptr(sums), s.shape[0], _ptr(out))
        else:
            f.argtypes = [C.c_int, C.c_int, _dp, C.c_int, _dp]
            n = f(int(D), int(F), _ptr(s), s.shape[0], _ptr(out))
        assert self._check(n) == N, (n, N)
        return out

    def sampled_strategy_fp(self, D, F, seed, num_iters=1024, max_depth=2, linear_update=True):
        """compute_sampled_strategy_recursive_to_leaf with fictitious play, zero net (reference only): dense [N_full, H, A]."""
        assert self.kind == "ref"
        A, H, Q = game_dims(D, F)
        N = (1 << A) - 1
        out = np.zeros((N, H, A), np.float64)
        f = self._f("sampled_strategy_fp")
        f.argtypes = [C.c_int] * 6 + [_dp]
        assert self._check(f(int(D), int(F), int(num_iters), int(max_depth), int(linear_update), int(seed), _ptr(out))) == N
        return out


if __name__ == "__main__":
    build_port()
    if len(sys.argv) > 1 and sys.argv[1] == "ref":
        build_ref()
