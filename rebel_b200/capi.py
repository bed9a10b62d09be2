"""ctypes binding of libcfrb200.so (include/cfrb200.h) — the same C ABI the C++ `rela` module links against.

There is no CPU fallback: importing works anywhere (so the symbol/ABI tests run without a GPU), but
``WaveSolver(...)`` raises unless the CUDA library is built (``__graft_entry__.build()``) and a device is present.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcfrb200.so")

NET_ZERO, NET_FP32, NET_TC_F16, NET_TC_F16X2 = 0, 1, 2, 3
SOLVER_CFR, SOLVER_FP = 0, 1
STATE_F64, STATE_F32 = 0, 1


class CfrbError(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [
        ("num_dice", C.c_int32), ("num_faces", C.c_int32), ("max_depth", C.c_int32), ("num_iters", C.c_int32),
        ("linear_update", C.c_int32), ("dcfr", C.c_int32),
        ("dcfr_alpha", C.c_double), ("dcfr_beta", C.c_double), ("dcfr_gamma", C.c_double),
        ("max_subgames", C.c_int32), ("device", C.c_int32), ("net_mode", C.c_int32), ("hidden", C.c_int32),
        ("state_dtype", C.c_int32), ("solver", C.c_int32), ("optimistic", C.c_int32),
    ]


_fp = C.POINTER(C.c_float)
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)
_lib = None


def lib():
    """Load the library (once) and declare prototypes.  Fails loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CfrbError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.cfrb_last_error.restype = C.c_char_p
    L.cfrb_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.cfrb_destroy.argtypes = [vp]
    for f in ("cfrb_num_actions", "cfrb_num_hands", "cfrb_query_size", "cfrb_max_nodes", "cfrb_iterations_done",
              "cfrb_sync"):
        getattr(L, f).argtypes = [vp]
    L.cfrb_unroll_tree.argtypes = [C.c_int32] * 5 + [_ip, C.c_int32]
    L.cfrb_tc_net_supported.argtypes = [C.c_int32] * 3
    L.cfrb_tree_template.argtypes = [vp, C.c_int32, C.c_int32, _ip, C.c_int32]
    L.cfrb_set_weights.argtypes = [vp, _fp, C.c_size_t, C.c_uint64]
    L.cfrb_weights_version.argtypes = [vp]
    L.cfrb_weights_version.restype = C.c_uint64
    L.cfrb_begin_wave.argtypes = [vp, C.c_int32, _ip, _ip, _dp, _ip]
    L.cfrb_run.argtypes = [vp, C.c_int32, vp]
    L.cfrb_reset_wave.argtypes = [vp, vp]
    L.cfrb_set_profiling.argtypes = [vp, C.c_int32]
    L.cfrb_fetch.argtypes = [vp] + [_dp] * 6
    L.cfrb_examples.argtypes = [vp, _fp, _fp]
    L.cfrb_table_stride.argtypes = [vp]
    L.cfrb_fetch_compact.argtypes = [vp, C.c_int32, _dp]
    L.cfrb_load_state.argtypes = [vp, _dp, _dp, _dp, _dp, _ip, C.c_int32]
    L.cfrb_debug_leaf_io.argtypes = [vp, _fp, _fp, _dp, C.c_int32]
    L.cfrb_exploitability.argtypes = [vp, _dp, _dp]
    L.cfrb_ev2.argtypes = [vp, _dp, _dp, _dp]
    L.cfrb_full_tree_nodes.argtypes = [vp]
    L.cfrb_to_leaf_exploitability.argtypes = [vp, _dp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), _dp]
    L.cfrb_to_leaf_bytes.argtypes = [C.c_int32] * 4
    L.cfrb_to_leaf_bytes.restype = C.c_int64
    L.cfrb_to_leaf_strategy.argtypes = [vp, _dp]
    L.cfrb_debug_to_leaf_free_cap.argtypes = [vp, C.c_int64]
    L.cfrb_regrets_reset.argtypes = [vp]
    L.cfrb_regrets_add.argtypes = [vp, _fp, C.c_int32]
    L.cfrb_regrets_add_current.argtypes = [vp]
    L.cfrb_regrets_fetch.argtypes = [vp, _dp, _dp, C.POINTER(C.c_int64)]
    L.cfrb_debug_net_taps.argtypes = [vp, _fp, _fp]
    L.cfrb_debug_net_trace.argtypes = [vp, C.POINTER(C.c_longlong), C.c_int]
    L.cfrb_kernel_launches.argtypes = [vp]
    L.cfrb_kernel_launches.restype = C.c_int64
    L.cfrb_wave_leaf_rows.argtypes = [vp]
    L.cfrb_wave_leaf_rows.restype = C.c_int64
    L.cfrb_last_run_ms.argtypes = [vp, _fp, _fp]
    L.cfrb_selfplay_create.argtypes = [vp, C.c_int32, C.POINTER(C.c_uint32), C.c_float, C.c_int32]
    L.cfrb_selfplay_wave.argtypes = [vp, vp, vp, C.c_int32, vp]
    L.cfrb_selfplay_wait_examples.argtypes = [vp]
    L.cfrb_selfplay_state.argtypes = [vp, _ip, _ip, _dp]
    L.cfrb_selfplay_export.argtypes = [vp, vp, C.c_size_t]
    L.cfrb_selfplay_export.restype = C.c_int64
    L.cfrb_selfplay_import.argtypes = [vp, C.c_char_p, C.c_size_t]
    L.cfrb_stream_wait.argtypes = [vp, vp]
    L.cfrb_debug_div_check.argtypes = [vp, C.c_uint64, C.c_int32, C.POINTER(C.c_uint64)]
    L.cfrb_debug_gelu_table.argtypes = [vp, C.c_int32, C.POINTER(C.c_uint16)]
    L.cfrb_wave_roots.argtypes = [vp, _ip, _ip, C.c_int32]
    L.cfrb_wave_order.argtypes = [vp, _ip, C.c_int32]
    L.cfrb_schedule_order.argtypes = [C.c_int32] * 4 + [_ip, _ip, C.POINTER(C.c_int64)]
    L.cfrb_debug_d2_grid.argtypes = [vp, C.c_int32]
    L.cfrb_mark.argtypes = [vp, C.c_int32, vp]
    L.cfrb_mark_elapsed_ms.argtypes = [vp, C.c_int32, C.c_int32, _fp]
    L.cfrb_l2_flush.argtypes = [vp, C.c_size_t, vp]
    L.cfrb_dev_alloc.argtypes = [C.c_int32, C.c_size_t, C.POINTER(vp)]
    L.cfrb_dev_free.argtypes = [C.c_int32, vp]
    L.cfrb_dev_to_host.argtypes = [C.c_int32, vp, vp, C.c_size_t]
    L.cfrb_rows_create.argtypes = [C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.POINTER(vp)]
    L.cfrb_rows_destroy.argtypes = [vp]
    L.cfrb_rows_device.argtypes = [vp]
    L.cfrb_rows_write.argtypes = [vp, C.c_int64, C.c_int32, vp, vp, C.c_int32, C.c_int32]
    L.cfrb_rows_read.argtypes = [vp, C.c_int64, C.c_int32, _fp, _fp]
    L.cfrb_rows_gather.argtypes = [vp, _ip, C.c_int32, vp, vp, C.c_int32, vp]
    L.cfrb_match_create.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_uint64, C.c_int32, C.POINTER(vp)]
    L.cfrb_match_run.argtypes = [vp, C.c_int32, vp]
    L.cfrb_match_results.argtypes = [vp, _fp, _ip, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.cfrb_match_trace.argtypes = [vp, C.c_int32, _ip, _dp, _ip, _dp, _ip]
    L.cfrb_match_destroy.argtypes = [vp]
    L.cfrb_match_create_lbr.argtypes = [vp, C.c_int32, C.c_int32, C.c_uint64, C.POINTER(vp)]
    L.cfrb_match_lbr_trace.argtypes = [vp, C.c_int32, _dp, _dp]
    L.cfrb_match_lbr_counts.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.cfrb_trainer_create.argtypes = [C.c_int32] * 4 + [C.POINTER(vp)]
    L.cfrb_trainer_destroy.argtypes = [vp]
    L.cfrb_trainer_num_params.argtypes = [vp]
    L.cfrb_trainer_num_params.restype = C.c_int64
    L.cfrb_trainer_set_state.argtypes = [vp, _fp, _fp, _fp, C.c_int64]
    L.cfrb_trainer_get_state.argtypes = [vp, _fp, _fp, _fp, C.POINTER(C.c_int64)]
    L.cfrb_trainer_step.argtypes = [vp, vp, vp, C.c_int32, C.c_double, C.c_double, C.c_int32, vp, vp]
    L.cfrb_trainer_loss.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, vp, vp]
    L.cfrb_trainer_last.argtypes = [vp, _fp, _fp]
    L.cfrb_trainer_debug_grads.argtypes = [vp, _fp]
    _lib = L
    return L


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _check(rc):
    if rc < 0:
        raise CfrbError(f"cfrb error {rc}: {lib().cfrb_last_error().decode()}")
    return rc


def unroll_tree(num_dice, num_faces, last_bid=-1, player_id=0, max_depth=1000000):
    """Host-only tree enumeration; rows = (last_bid, player_id, children_begin, children_end, parent, depth)."""
    cap = 1 << 16
    out = np.zeros((cap, 6), np.int32)
    n = _check(lib().cfrb_unroll_tree(num_dice, num_faces, last_bid, player_id, max_depth, _p(out, _ip), cap))
    return out[:n].copy()


def schedule_order(num_dice, num_faces, last_bid, max_depth=2):
    """Host-only: (order, cost) — the order in which the depth-2 CFR kernel starts subgames rooted at last_bid (wave positions,
    costliest first, stable) and each subgame's schedule cost."""
    lb = np.ascontiguousarray(last_bid, np.int32)
    order = np.zeros(lb.size, np.int32)
    cost = np.zeros(lb.size, np.int64)
    _check(lib().cfrb_schedule_order(num_dice, num_faces, max_depth, lb.size, _p(lb, _ip), _p(order, _ip),
                                     cost.ctypes.data_as(C.POINTER(C.c_int64))))
    return order, cost


def to_leaf_bytes(num_dice, num_faces, max_depth, max_subgames):
    """Host-only: device bytes WaveSolver.to_leaf_exploitability needs beyond a handle of these sizes (full tree, best-response
    scratch, the walk's largest levels)."""
    return _check(lib().cfrb_to_leaf_bytes(num_dice, num_faces, max_depth, max_subgames))


def tc_net_supported(num_dice, num_faces, hidden=256):
    """Host-only: does a tensor-core value net (NET_TC_F16 / NET_TC_F16X2) fit this game?  Otherwise NET_FP32 serves it."""
    return bool(lib().cfrb_tc_net_supported(num_dice, num_faces, hidden))


class WaveSolver:
    """K concurrent CFR subgames on one GPU.  Mirrors build_solver + ISubgameSolver (subgame_solving.h:60-134)
    for a whole wave: begin() ~ constructor, run() ~ step/multistep, getters ~ get_*."""

    def __init__(self, num_dice, num_faces, max_subgames, max_depth=2, num_iters=1024, linear_update=True, dcfr=False,
                 dcfr_alpha=0.0, dcfr_beta=0.0, dcfr_gamma=0.0, net_mode=NET_FP32, hidden=256, device=0,
                 state_dtype=STATE_F64, solver=SOLVER_CFR, optimistic=False):
        L = lib()
        self.cfg = Config(num_dice, num_faces, max_depth, num_iters, int(linear_update), int(dcfr), dcfr_alpha, dcfr_beta,
                          dcfr_gamma, max_subgames, device, net_mode, hidden, state_dtype, int(solver), int(optimistic))
        self._h = C.c_void_p()
        _check(L.cfrb_create(C.byref(self.cfg), C.byref(self._h)))
        self.A = L.cfrb_num_actions(self._h)
        self.H = L.cfrb_num_hands(self._h)
        self.Q = L.cfrb_query_size(self._h)
        self.Nmax = L.cfrb_max_nodes(self._h)
        self.n = 0

    def close(self):
        if self._h:
            lib().cfrb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def tree(self, last_bid=-1, player_id=0):
        out = np.zeros((self.Nmax, 6), np.int32)
        n = _check(lib().cfrb_tree_template(self._h, last_bid, player_id, _p(out, _ip), self.Nmax))
        return out[:n].copy()

    def set_weights(self, flat, version=0):
        w = np.ascontiguousarray(flat, np.float32)
        _check(lib().cfrb_set_weights(self._h, _p(w, _fp), w.size, version))

    def begin(self, last_bid, player_id, beliefs, act_iteration=None):
        lb = np.ascontiguousarray(last_bid, np.int32)
        pl = np.ascontiguousarray(player_id, np.int32)
        b = np.ascontiguousarray(beliefs, np.float64)
        n = lb.shape[0]
        assert pl.shape == (n,) and b.shape == (n, 2, self.H), (pl.shape, b.shape)
        act = None if act_iteration is None else np.ascontiguousarray(act_iteration, np.int32)
        _check(lib().cfrb_begin_wave(self._h, n, _p(lb, _ip), _p(pl, _ip), _p(b, _dp), _p(act, _ip)))
        self.n = n

    def reset(self, stream=None):
        _check(lib().cfrb_reset_wave(self._h, C.c_void_p(stream) if stream else None))

    def set_profiling(self, on):
        _check(lib().cfrb_set_profiling(self._h, int(on)))

    def run(self, iters, stream=None):
        _check(lib().cfrb_run(self._h, iters, C.c_void_p(stream) if stream else None))

    def sync(self):
        _check(lib().cfrb_sync(self._h))

    @property
    def iterations_done(self):
        return lib().cfrb_iterations_done(self._h)

    def fetch(self, want=("root_means", "last", "avg")):
        """dict of: root_means [n,2,H]; snapshot/last/avg/sum/regrets dense [n,Nmax,H,A]."""
        n = self.n
        bufs = {}
        if "root_means" in want:
            bufs["root_means"] = np.zeros((n, 2, self.H), np.float64)
        for k in ("snapshot", "last", "avg", "sum", "regrets"):
            if k in want:
                bufs[k] = np.zeros((n, self.Nmax, self.H, self.A), np.float64)
        g = lambda k: _p(bufs.get(k), _dp)
        _check(lib().cfrb_fetch(self._h, g("root_means"), g("snapshot"), g("last"), g("avg"), g("sum"), g("regrets")))
        return bufs

    def fetch_compact(self, which="snapshot"):
        """[n, table_stride] fp64; entry (child - 1) * H + hand = value of (parent, hand, action to child)."""
        stride = lib().cfrb_table_stride(self._h)
        out = np.zeros((self.n, stride), np.float64)
        _check(lib().cfrb_fetch_compact(self._h, {"snapshot": 0, "last": 1, "sum": 2, "regrets": 3}[which], _p(out, _dp)))
        return out

    def examples(self):
        q = np.zeros((self.n, 2, self.Q), np.float32)
        v = np.zeros((self.n, 2, self.H), np.float32)
        _check(lib().cfrb_examples(self._h, _p(q, _fp), _p(v, _fp)))
        return q, v

    def load_state(self, regrets=None, last=None, sum=None, root_means=None, num_steps=None, iterations_done=0):
        c = lambda a, t: None if a is None else np.ascontiguousarray(a, t)
        r, l, s, m, st = c(regrets, np.float64), c(last, np.float64), c(sum, np.float64), c(root_means, np.float64), \
            c(num_steps, np.int32)
        _check(lib().cfrb_load_state(self._h, _p(r, _dp), _p(l, _dp), _p(s, _dp), _p(m, _dp), _p(st, _ip), iterations_done))

    def leaf_io(self):
        rows = lib().cfrb_wave_leaf_rows(self._h)
        q = np.zeros((max(rows, 1), self.Q), np.float32)
        o = np.zeros((max(rows, 1), self.H), np.float32)
        s = np.zeros(max(rows, 1), np.float64)
        _check(lib().cfrb_debug_leaf_io(self._h, _p(q, _fp), _p(o, _fp), _p(s, _dp), rows))
        return q[:rows], o[:rows], s[:rows]

    def net_taps(self):
        d1 = np.zeros((128, 256), np.float32)
        d2 = np.zeros((128, 256), np.float32)
        _check(lib().cfrb_debug_net_taps(self._h, _p(d1, _fp), _p(d2, _fp)))
        return d1, d2

    def net_trace(self):
        t = np.zeros(2048, np.int64)
        _check(lib().cfrb_debug_net_trace(self._h, t.ctypes.data_as(C.POINTER(C.c_longlong)), 2048))
        return t

    def exploitability(self, full_strategy):
        s = np.ascontiguousarray(full_strategy, np.float64)
        out = np.zeros(2, np.float64)
        _check(lib().cfrb_exploitability(self._h, _p(s, _dp), _p(out, _dp)))
        return out

    def to_leaf_exploitability(self):
        """Exploitability of the recursive to-leaf average policy of this handle (its weights and solver settings), walked level by
        level in waves of max_subgames on the device: dict of br [2], exploitability, subgames, subgame_iters, walk_seconds,
        br_seconds.  Replaces the handle's wave."""
        br, secs = np.zeros(2, np.float64), np.zeros(2, np.float64)
        sg, it = C.c_int64(0), C.c_int64(0)
        _check(lib().cfrb_to_leaf_exploitability(self._h, _p(br, _dp), C.byref(sg), C.byref(it), _p(secs, _dp)))
        return {"br": br, "exploitability": (br[0] + br[1]) / 2, "subgames": sg.value, "subgame_iters": it.value,
                "walk_seconds": float(secs[0]), "br_seconds": float(secs[1])}

    def to_leaf_strategy(self):
        """The compact full-tree strategy [N_full - 1, H] the last to_leaf_exploitability filled (entry [child - 1, hand])."""
        n = (1 << self.A) - 1                    # the full Liar's Dice tree
        out = np.zeros((max(n - 1, 1), self.H), np.float64)
        _check(lib().cfrb_to_leaf_strategy(self._h, _p(out, _dp)))
        return out

    def debug_to_leaf_free_cap(self, nbytes):
        """Test aid: to_leaf_exploitability sees at most nbytes free device bytes (0 = the device's own figure)."""
        _check(lib().cfrb_debug_to_leaf_free_cap(self._h, int(nbytes)))

    @property
    def kernel_launches(self):
        return lib().cfrb_kernel_launches(self._h)

    @property
    def leaf_rows(self):
        return lib().cfrb_wave_leaf_rows(self._h)

    # ---- device-resident self-play (cfrb_selfplay_*)
    def selfplay_create(self, seeds, random_action_prob=0.25, sample_leaf=True):
        s = np.ascontiguousarray(seeds, np.uint32)
        _check(lib().cfrb_selfplay_create(self._h, s.size, s.ctypes.data_as(C.POINTER(C.c_uint32)), random_action_prob, int(sample_leaf)))
        self.n = s.size
        self._sp_bufs = None

    def selfplay_wave(self, start_next=True, keep_examples=False, stream=None):
        """Finish the pending wave and (optionally) start the next one, asynchronously.  keep_examples: the finished wave's
        examples go to a device buffer owned by this object; examples() then copies them to the host."""
        q = v = None
        if keep_examples:
            if self._sp_bufs is None:
                a, b = C.c_void_p(), C.c_void_p()
                _check(lib().cfrb_dev_alloc(self.cfg.device, self.n * 2 * self.Q * 4, C.byref(a)))
                _check(lib().cfrb_dev_alloc(self.cfg.device, self.n * 2 * self.H * 4, C.byref(b)))
                self._sp_bufs = (a, b)
            q, v = self._sp_bufs
        return _check(lib().cfrb_selfplay_wave(self._h, q, v, int(start_next), C.c_void_p(stream) if stream else None))

    def selfplay_examples(self):
        lib().cfrb_selfplay_wait_examples(self._h)
        q = np.zeros((self.n, 2, self.Q), np.float32)
        v = np.zeros((self.n, 2, self.H), np.float32)
        _check(lib().cfrb_dev_to_host(self.cfg.device, q.ctypes.data_as(C.c_void_p), self._sp_bufs[0], q.nbytes))
        _check(lib().cfrb_dev_to_host(self.cfg.device, v.ctypes.data_as(C.c_void_p), self._sp_bufs[1], v.nbytes))
        return q, v

    def selfplay_state(self):
        lb = np.zeros(self.n, np.int32); pl = np.zeros(self.n, np.int32); b = np.zeros((self.n, 2, self.H), np.float64)
        _check(lib().cfrb_selfplay_state(self._h, _p(lb, _ip), _p(pl, _ip), _p(b, _dp)))
        return lb, pl, b

    def selfplay_export(self):
        """The session's image (bytes): every game's state and random stream.  Needs a drained session (no pending wave)."""
        n = _check(lib().cfrb_selfplay_export(self._h, None, 0))
        buf = C.create_string_buffer(n)
        _check(lib().cfrb_selfplay_export(self._h, buf, n))
        return buf.raw

    def selfplay_import(self, image):
        """Install an image of selfplay_export into this handle's session (same game, n_games, sampling parameters)."""
        image = bytes(image)
        _check(lib().cfrb_selfplay_import(self._h, image, len(image)))

    def gelu_table(self, what):
        """fp16 -> fp16 table of tanh.approx.f16x2 (what=0) / of the epilogue's GELU from hy = y/2, packed-half (what=1) or fp32-tanh
        (what=2) evaluation, as float16 arrays (x, f(x))."""
        out = np.zeros(65536, np.uint16)
        _check(lib().cfrb_debug_gelu_table(self._h, what, out.ctypes.data_as(C.POINTER(C.c_uint16))))
        return np.arange(65536, dtype=np.uint16).view(np.float16), out.view(np.float16)

    def div_check(self, seed, blocks):
        bad = C.c_uint64(0)
        _check(lib().cfrb_debug_div_check(self._h, seed, blocks, C.byref(bad)))
        return bad.value

    def wave_roots(self):
        lb = np.zeros(self.n, np.int32); pl = np.zeros(self.n, np.int32)
        n = _check(lib().cfrb_wave_roots(self._h, _p(lb, _ip), _p(pl, _ip), self.n))
        return lb[:n], pl[:n]

    def wave_order(self):
        """The order in which the depth-2 CFR kernel starts the current wave's subgames (wave positions)."""
        out = np.zeros(self.n, np.int32)
        n = _check(lib().cfrb_wave_order(self._h, _p(out, _ip), self.n))
        return out[:n]

    def debug_d2_grid(self, max_ctas):
        """Test aid: run the depth-2 CFR kernel on at most max_ctas CTAs (0 = no cap); returns the CTAs resident at once."""
        return _check(lib().cfrb_debug_d2_grid(self._h, int(max_ctas)))

    def wait_examples(self):
        _check(lib().cfrb_selfplay_wait_examples(self._h))

    def mark(self, slot, stream=None):
        _check(lib().cfrb_mark(self._h, slot, C.c_void_p(stream) if stream else None))

    def elapsed_ms(self, a, b):
        ms = C.c_float(0)
        _check(lib().cfrb_mark_elapsed_ms(self._h, a, b, C.byref(ms)))
        return ms.value

    def l2_flush(self, nbytes=256 << 20, stream=None):
        _check(lib().cfrb_l2_flush(self._h, nbytes, C.c_void_p(stream) if stream else None))

    def last_run_ms(self):
        a, b = C.c_float(0), C.c_float(0)
        _check(lib().cfrb_last_run_ms(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value


MATCH_AVERAGE, MATCH_SAMPLED = 0, 1
MATCH_TRACE_GAMES = 256


class Match:
    """A head-to-head match between the agents of two WaveSolvers (cfrb_match_*): n_games games, n_slots at a time."""

    def __init__(self, a, b, n_slots, n_games, seed=0, policy=MATCH_SAMPLED):
        self.a, self.b, self.G = a, b, n_games
        self._m = C.c_void_p()
        _check(lib().cfrb_match_create(a._h, b._h, n_slots, n_games, seed, policy, C.byref(self._m)))

    def close(self):
        if self._m:
            lib().cfrb_match_destroy(self._m)
            self._m = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def run(self, max_rounds=8, stream=None):
        """Enqueue rounds; 0 once every game has finished."""
        return _check(lib().cfrb_match_run(self._m, max_rounds, C.c_void_p(stream) if stream else None))

    def play(self):
        while self.run() > 0:
            pass
        return self.results()

    def results(self):
        pay = np.zeros(self.G, np.float32)
        plies = np.zeros(self.G, np.int32)
        solves, iters = C.c_int64(0), C.c_int64(0)
        _check(lib().cfrb_match_results(self._m, _p(pay, _fp), _p(plies, _ip), C.byref(solves), C.byref(iters)))
        return {"payoff_a": pay, "plies": plies, "solves": solves.value, "subgame_iters": iters.value}

    def trace(self, game):
        """dict: plies [P, 6] (agent, last bid, player, hand, action, round), prob [P], act_iteration [R, 2], root_beliefs [R, 2, 2, H]."""
        A, H = self.a.A, self.a.H
        rec = np.zeros((A, 6), np.int32)
        prob = np.zeros(A, np.float64)
        act = np.zeros((A, 2), np.int32)
        bel = np.zeros((A, 2, 2, H), np.float64)
        nr = C.c_int32(0)
        n = _check(lib().cfrb_match_trace(self._m, game, _p(rec, _ip), _p(prob, _dp), _p(act, _ip), _p(bel, _dp), C.byref(nr)))
        r = nr.value
        return {"plies": rec[:n], "prob": prob[:n], "act_iteration": act[:r], "root_beliefs": bel[:r]}


class LbrMatch(Match):
    """Local best response against the agent of one WaveSolver (cfrb_match_create_lbr): n_games games, n_slots at a time, at
    most the solver's max_subgames subgames per round.  results()["payoff_a"] is the agent's payoff; in trace() agent 1 is LBR."""

    def __init__(self, agent, n_slots, n_games, seed=0):
        self.a, self.b, self.G = agent, None, n_games
        self._m = C.c_void_p()
        _check(lib().cfrb_match_create_lbr(agent._h, n_slots, n_games, seed, C.byref(self._m)))

    def results(self):
        r = super().results()
        w, d = C.c_int64(0), C.c_int64(0)
        _check(lib().cfrb_match_lbr_counts(self._m, C.byref(w), C.byref(d)))
        r["whatif_solves"], r["deferred_slot_rounds"] = w.value, d.value
        return r

    def lbr_trace(self, game):
        """dict: values [P, A] (value of each of LBR's actions at ply i, NaN where illegal or on the agent's plies), beliefs [P, H]
        (LBR's belief over the agent's hand before the decision)."""
        A, H = self.a.A, self.a.H
        val = np.zeros((A, A), np.float64)
        bel = np.zeros((A, H), np.float64)
        n = _check(lib().cfrb_match_lbr_trace(self._m, game, _p(val, _dp), _p(bel, _dp)))
        return {"values": val[:n], "beliefs": bel[:n]}
