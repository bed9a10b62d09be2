"""Training of the value net on the GPU: ``Net2Trainer`` runs the reference trainer's optimisation step (cfvpy/selfplay.py:409-438:
forward, huber / mse loss, backward, clip_grad_norm_, Adam) for Net2(n_hidden=256, n_layers=2, use_layer_norm=True) as CUDA
kernels of libcfrb200 (cfrb_trainer_*, include/cfrb200.h), in fp32 and deterministically.

    tr = Net2Trainer(1, 6, "cuda:0")
    batch, _ = replay.sample(512, "cuda:0")          # rela.ValuePrioritizedReplay
    loss, grad_norm = tr.step(batch.query, batch.values)
    locker.update_model(tr.net())                     # rela.ModelLocker: the generator loops pick the weights up

A step is enqueued on the current torch stream of the trainer's device and returns device tensors: nothing synchronises until
the caller reads them.  ``optimizer_state()`` / ``load_optimizer_state()`` use the layout of ``torch.optim.Adam.state_dict()``, so a
run can move between torch and this trainer in either direction.
"""
import ctypes as C

import numpy as np
import torch

from rebel_b200 import capi
from rebel_b200.models import FLAT_ORDER, Net2, flatten_state_dict, input_size, make_selfplay_net, output_size

LOSSES = {"huber": 0, "mse": 1}
ADAM_DEFAULTS = dict(betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, maximize=False)


def check_state_dict(sd, num_dice, num_faces):
    """Flat fp32 weights of a Net2(n_hidden=256, n_layers=2, use_layer_norm=True) state_dict for this game, or ValueError: the
    rules of flatten_state_dict / ModelLocker plus the game's input and output widths."""
    flat = flatten_state_dict(sd)
    Q, H = input_size(num_faces, num_dice), output_size(num_faces, num_dice)
    if tuple(sd["body.0.weight"].shape) != (256, Q):
        raise ValueError(f"body.0.weight is {tuple(sd['body.0.weight'].shape)}, the {num_dice}x{num_faces}f net needs (256, {Q})")
    if tuple(sd["output.weight"].shape) != (H, 256):
        raise ValueError(f"output.weight is {tuple(sd['output.weight'].shape)}, the {num_dice}x{num_faces}f net needs ({H}, 256)")
    return flat


class Net2Trainer:
    """Parameters, Adam moments, step count and scratch of one value net on one GPU.

    state_dict: the initial weights (default: make_selfplay_net(num_dice, num_faces, seed)).  It is checked before the device
    is touched.  lr, grad_clip (0 = no clipping) and loss ("huber" / "mse") are the reference trainer's cfg.optimizer.kwargs.lr,
    cfg.grad_clip and cfg.loss; lr may be changed between steps (the halving schedule)."""

    def __init__(self, num_dice, num_faces, device="cuda:0", max_batch=512, lr=3e-4, grad_clip=5.0, loss="huber",
                 state_dict=None, seed=0):
        if loss not in LOSSES:
            raise ValueError(f"loss must be one of {sorted(LOSSES)}, got {loss!r}")
        if max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self.num_dice, self.num_faces = num_dice, num_faces
        self.Q, self.H = input_size(num_faces, num_dice), output_size(num_faces, num_dice)
        self.max_batch, self.lr, self.grad_clip, self.loss_name = int(max_batch), float(lr), float(grad_clip), loss
        if state_dict is None:
            state_dict = make_selfplay_net(num_dice, num_faces, seed).state_dict()
        flat = check_state_dict(state_dict, num_dice, num_faces)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"Net2Trainer runs on a CUDA device, got {device!r}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._t = C.c_void_p()
        capi._check(capi.lib().cfrb_trainer_create(self.device.index, num_dice, num_faces, self.max_batch, C.byref(self._t)))
        self.P = capi.lib().cfrb_trainer_num_params(self._t)
        self._set(flat, None, None, 0)
        self.last_row_loss = None

    def close(self):
        if self._t:
            capi.lib().cfrb_trainer_destroy(self._t)
            self._t = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- state
    def _set(self, flat, m, v, step):
        c = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
        flat, m, v = c(flat), c(m), c(v)
        for name, a in (("params", flat), ("exp_avg", m), ("exp_avg_sq", v)):
            if a is not None and a.size != self.P:
                raise ValueError(f"{name} has {a.size} floats, the trainer holds {self.P}")
        capi._check(capi.lib().cfrb_trainer_set_state(self._t, capi._p(flat, capi._fp), capi._p(m, capi._fp), capi._p(v, capi._fp),
                                                       int(step)))

    def get_state(self):
        """(params, exp_avg, exp_avg_sq) flat fp32 numpy arrays in FLAT_ORDER and the Adam step count.  Synchronises."""
        p, m, v = (np.zeros(self.P, np.float32) for _ in range(3))
        s = C.c_int64(0)
        capi._check(capi.lib().cfrb_trainer_get_state(self._t, capi._p(p, capi._fp), capi._p(m, capi._fp), capi._p(v, capi._fp),
                                                       C.byref(s)))
        return p, m, v, s.value

    def set_state(self, params, exp_avg=None, exp_avg_sq=None, step=0):
        self._set(params, exp_avg, exp_avg_sq, step)

    def load_state_dict(self, sd):
        """Install the weights of a Net2 state_dict; the Adam state is kept."""
        flat = check_state_dict(sd, self.num_dice, self.num_faces)
        _, m, v, step = self.get_state()
        self._set(flat, m, v, step)

    def _split(self, flat):
        out, off = {}, 0
        shapes = {k: tuple(t.shape) for k, t in self._template().state_dict().items()}
        for k in FLAT_ORDER:
            n = int(np.prod(shapes[k]))
            out[k] = torch.from_numpy(flat[off:off + n].copy()).reshape(shapes[k])
            off += n
        return out

    def _template(self):
        return Net2(num_faces=self.num_faces, num_dice=self.num_dice, n_hidden=256, n_layers=2, use_layer_norm=True)

    def state_dict(self):
        return self._split(self.get_state()[0])

    def net(self):
        """A rebel_b200.models.Net2 (on the CPU, eval mode) holding the current weights: for torch.save(net.state_dict()),
        torch.jit.script and ModelLocker.update_model."""
        net = self._template()
        net.load_state_dict(self.state_dict())
        return net.eval()

    def grads(self):
        """Test aid: the gradients of the most recent step after clipping, by parameter name.  Synchronises."""
        g = np.zeros(self.P, np.float32)
        capi._check(capi.lib().cfrb_trainer_debug_grads(self._t, capi._p(g, capi._fp)))
        return self._split(g)

    def optimizer_state(self):
        """The Adam state in the layout of torch.optim.Adam(net.parameters(), lr).state_dict()."""
        p, m, v, step = self.get_state()
        net = self._template()
        opt = torch.optim.Adam(net.parameters(), lr=self.lr)
        if step > 0:
            ms, vs = self._split(m), self._split(v)
            for k, prm in zip(FLAT_ORDER, net.parameters()):
                opt.state[prm] = {"step": torch.tensor(float(step)), "exp_avg": ms[k], "exp_avg_sq": vs[k]}
        return opt.state_dict()

    def load_optimizer_state(self, osd):
        """Install the Adam state (and lr) of a torch.optim.Adam state_dict over the parameters of a Net2 of this game."""
        groups = osd["param_groups"]
        if len(groups) != 1 or len(groups[0]["params"]) != len(FLAT_ORDER):
            raise ValueError("expected one parameter group over the 10 parameters of Net2(n_layers=2, use_layer_norm=True)")
        g = groups[0]
        for k, want in ADAM_DEFAULTS.items():
            got = g.get(k, want)
            if (tuple(got) if isinstance(got, (list, tuple)) else got) != want:
                raise ValueError(f"Adam {k}={got!r}: the trainer implements {k}={want!r} only")
        p, _, _, _ = self.get_state()
        state = osd["state"]
        if not state:
            self._set(p, None, None, 0)
        else:
            shapes = {k: tuple(t.shape) for k, t in self._template().state_dict().items()}
            ms, vs, steps = [], [], set()
            for k, idx in zip(FLAT_ORDER, g["params"]):
                s = state[idx]
                if tuple(s["exp_avg"].shape) != shapes[k]:
                    raise ValueError(f"exp_avg of {k} is {tuple(s['exp_avg'].shape)}, expected {shapes[k]}")
                ms.append(s["exp_avg"].detach().float().cpu().reshape(-1))
                vs.append(s["exp_avg_sq"].detach().float().cpu().reshape(-1))
                steps.add(int(float(s["step"])))
            if len(steps) != 1:
                raise ValueError(f"parameters have different Adam step counts {sorted(steps)}")
            self._set(p, torch.cat(ms).numpy(), torch.cat(vs).numpy(), steps.pop())
        self.lr = float(g["lr"])

    @property
    def steps(self):
        return self.get_state()[3]

    # ---- compute
    def _batch(self, query, values):
        for name, t, w in (("query", query, self.Q), ("values", values, self.H)):
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{name} must be a torch tensor")
            if t.device != self.device:
                raise ValueError(f"{name} is on device {t.device}, the trainer is on {self.device}")
            if t.dtype != torch.float32:
                raise ValueError(f"{name} must be float32, got {t.dtype}")
            if t.dim() != 2 or t.shape[1] != w:
                raise ValueError(f"{name} has shape {tuple(t.shape)}, expected (n, {w}) for {self.num_dice}x{self.num_faces}f")
        n = query.shape[0]
        if values.shape[0] != n:
            raise ValueError(f"query has {n} rows, values {values.shape[0]}")
        if not 1 <= n <= self.max_batch:
            raise ValueError(f"batch of {n} rows, the trainer takes 1 .. max_batch = {self.max_batch}")
        return query.contiguous(), values.contiguous(), n

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def step(self, query, values, lr=None):
        """One optimisation step on the batch; returns (loss, pre-clip grad norm) as 0-d device tensors.  The per-example losses
        (mean over the outputs) are left in self.last_row_loss [n]."""
        q, v, n = self._batch(query, values)
        out = torch.empty(2 + n, dtype=torch.float32, device=self.device)
        capi._check(capi.lib().cfrb_trainer_step(self._t, C.c_void_p(q.data_ptr()), C.c_void_p(v.data_ptr()), n,
                                                 self.lr if lr is None else float(lr), self.grad_clip, LOSSES[self.loss_name],
                                                 self._stream(), C.c_void_p(out.data_ptr())))
        self.last_row_loss = out[2:]
        return out[0], out[1]

    def loss(self, query, values):
        """Loss of the current net on a batch (forward only) as a 0-d device tensor."""
        q, v, n = self._batch(query, values)
        out = torch.empty(2 + n, dtype=torch.float32, device=self.device)
        capi._check(capi.lib().cfrb_trainer_loss(self._t, C.c_void_p(q.data_ptr()), C.c_void_p(v.data_ptr()), n,
                                                 LOSSES[self.loss_name], self._stream(), C.c_void_p(out.data_ptr())))
        return out[0]

    def last(self):
        """(loss, grad norm) of the most recent step as Python floats.  Synchronises."""
        a, b = C.c_float(0), C.c_float(0)
        capi._check(capi.lib().cfrb_trainer_last(self._t, C.byref(a), C.byref(b)))
        return a.value, b.value
