"""`actor` / `critic` with the reference's constructor signatures, parameter names and
state_dict keys (models.py:16-41, 52-88), backed by ONE flat fp32 device buffer per network.

The flat buffer (layout from `d4pg_actor_layout` / `d4pg_critic_layout`) is what the CUDA
learner, the fused Adam/Polyak kernel and the gradient all-reduce operate on; the
`fc1/fc2/fc2_2/fc3` `nn.Parameter`s are views into it, so `state_dict()` /
`load_state_dict()` / `torch.save` interchange `.pth` files with the reference
(main.py:367-368).  `forward` runs the sm_90a kernels through the C ABI; there is no
eager/CPU fallback -- on a box without a GPU the modules can be built and (de)serialised
but `forward` raises.
"""
import math

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib
from .utils import default_device

HIDDEN = _lib.HIDDEN
_LAYER_NAMES = ("fc1", "fc2", "fc2_2", "fc3")


def fanin_init(size, fanin=None):
    """N(0, 1/sqrt(size[0])) -- size[0] is out_features (models.py:6-9)."""
    fanin = fanin or size[0]
    return torch.empty(size).normal_(0.0, 1.0 / np.sqrt(fanin))


def _layout_py(dims):
    """Pure-Python mirror of the C layout rule (d4pg_*_layout): weight rows are padded to a pitch
    of 4 floats (16-B rows, TMA / float4 addressable), every tensor starts 4-float aligned."""
    offs, sizes, pitches, off = [], [], [], 0
    for fin, fout in dims:
        pitch = (fin + 3) & ~3
        pitches.append(pitch)
        for n in (pitch * fout, fout):
            offs.append(off)
            sizes.append(n)
            off = (off + n + 3) & ~3
    return offs, sizes, off, pitches


class _LinearView(nn.Module):
    """Holds `weight` [out,in] and `bias` [out] as views of the owner's flat buffer."""

    def __init__(self, in_features, out_features):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(0), requires_grad=True)
        self.bias = nn.Parameter(torch.empty(0), requires_grad=True)


class _FlatNet(nn.Module):
    precision = 0        # 0 fp32 FFMA, 1 3xTF32 wgmma, 2 TF32 wgmma, 3 bf16 wgmma (set per instance to switch forward())
    # True: with grad mode on and a parameter or input requiring grad, forward() records an autograd node whose backward
    # runs d4pg_*_backward (loss.backward() fills .grad -- kept in the flat gradient buffer -- and d input).
    # False: forward() returns a plain tensor.
    differentiable = False
    # ObsNormalizer (obs_norm.py) or None: when set, the `state` input goes through it before fc1 (a DDPG with obs_norm
    # attaches its normalizer to all four networks); the critic's action input is never normalized
    obs_normalizer = None

    def __init__(self, dims, device=None, empty=False):
        super().__init__()
        self._dims = list(dims)
        self._offsets, self._sizes, self._total, self._pitch = _layout_py(self._dims)
        self._device = torch.device(device) if device is not None else default_device()
        # empty=True: the buffer is left unwritten for a kernel that writes every float of it, pads included
        self._flat = (torch.empty if empty else torch.zeros)(self._total, dtype=torch.float32, device=self._device)
        self._flat_grad = None
        for name, (fin, fout) in zip(_LAYER_NAMES, self._dims):
            setattr(self, name, _LinearView(fin, fout))
        self._bind()

    # ---- flat storage plumbing --------------------------------------------------------
    def _views(self, flat):
        out = []
        for i, (fin, fout) in enumerate(self._dims):
            ow, ob, pitch = self._offsets[2 * i], self._offsets[2 * i + 1], self._pitch[i]
            # [out, in] view with a padded row pitch; the pad columns are never exposed
            out.append((flat[ow:ow + pitch * fout].view(fout, pitch)[:, :fin], flat[ob:ob + fout]))
        return out

    def _bind(self):
        for name, (w, b) in zip(_LAYER_NAMES, self._views(self._flat)):
            layer = getattr(self, name)
            layer.weight.data = w
            layer.bias.data = b
            layer.weight._d4pg_owner = self
            layer.bias._d4pg_owner = self
        if self._flat_grad is not None:
            self._bind_grads()

    def _bind_grads(self):
        for name, (w, b) in zip(_LAYER_NAMES, self._views(self._flat_grad)):
            layer = getattr(self, name)
            layer.weight.grad = w
            layer.bias.grad = b

    def flat_params(self):
        return self._flat

    def named_grad_views(self):
        """{state_dict key: view into the flat gradient buffer} (same shapes as the parameters)."""
        out = {}
        for name, (w, b) in zip(_LAYER_NAMES, self._views(self.flat_grads())):
            out[name + ".weight"], out[name + ".bias"] = w, b
        return out

    def flat_grads(self):
        """Flat gradient buffer (allocated on first use); `.grad` of every parameter views it.  A `.grad` that autograd
        put elsewhere (a parameter used outside this module's forward, or one reset to None) is taken over: its values
        are copied into the buffer (None counts as zero) and `.grad` views the buffer again."""
        if self._flat_grad is None:
            self._flat_grad = torch.zeros_like(self._flat)
        self._adopt_grads()
        return self._flat_grad

    def _grad_in_flat(self, g):
        f = self._flat_grad
        return (f is not None and g is not None and g.device == f.device
                and f.data_ptr() <= g.data_ptr() < f.data_ptr() + f.numel() * f.element_size())

    def _adopt_grads(self):
        for name, (w, b) in zip(_LAYER_NAMES, self._views(self._flat_grad)):
            layer = getattr(self, name)
            for p, view in ((layer.weight, w), (layer.bias, b)):
                if self._grad_in_flat(p.grad):
                    continue
                with torch.no_grad():
                    if p.grad is None:
                        view.zero_()
                    else:
                        view.copy_(p.grad)
                p.grad = view

    def adopt_flat(self, flat):
        """Alias another network's flat parameter storage (local == global model,
        what ddpg.py:104-108 / ddpg.py:118-120 establish in the single-worker reference)."""
        assert flat.numel() == self._total and flat.dtype == torch.float32
        self._flat = flat
        self._device = flat.device
        self._bind()

    def _apply(self, fn, *args, **kwargs):
        # .to()/.cuda()/.cpu(): move the flat buffer, then re-create the views
        new_flat = fn(self._flat)
        self._flat = new_flat.contiguous()
        self._device = self._flat.device
        if self._flat_grad is not None:
            self._flat_grad = fn(self._flat_grad).contiguous()
        self._bind()
        return self

    def load_state_dict(self, state_dict, strict=True, assign=False):
        # the copies go through the parameters, whose version counters are their own (a `.data` assignment does not
        # share the flat buffer's), so the flat buffer's counter -- which DDPG.train() watches to re-pack the learner's
        # weight images -- is advanced here
        out = super().load_state_dict(state_dict, strict=strict, assign=assign)
        torch.autograd.graph.increment_version(self._flat)
        return out

    def share_memory(self):
        # CUDA storage is already visible to every stream of the process; the reference's
        # cross-process sharing (ddpg.py:96-98) is replaced by NCCL data parallelism.
        return self

    def zero_grad(self, set_to_none=False):
        if self._flat_grad is not None:
            self._flat_grad.zero_()
        for p in self._param_list():          # a .grad outside the flat buffer (see flat_grads)
            if p.grad is not None and not self._grad_in_flat(p.grad):
                if set_to_none:
                    p.grad = None
                else:
                    with torch.no_grad():
                        p.grad.zero_()

    def _workspace(self, B):
        need = 3 * B * HIDDEN
        ws = getattr(self, "_ws", None)
        if ws is None or ws.numel() < need or ws.device != self._flat.device:
            ws = torch.empty(need, dtype=torch.float32, device=self._flat.device)
            self._ws = ws
        return ws

    def _input(self, x, width, grad):
        """An input as the kernels take it: [B, width] contiguous fp32 on this module's device.  With `grad` the
        conversion stays on the autograd graph (no detach)."""
        if grad and self._flat.device.type != "cuda":
            raise _lib.D4PGError("the D4PG kernels run only on a CUDA device (sm_90a); this module lives on %s"
                                 % self._flat.device)
        if not torch.is_tensor(x):
            x = torch.as_tensor(np.asarray(x))
        x = (x if grad else x.detach()).to(device=self._flat.device, dtype=torch.float32)
        if x.dim() == 1:
            x = x.view(1, -1)
        assert x.shape[1] == width, "expected input width %d, got %s" % (width, tuple(x.shape))
        return x.contiguous()

    def _state_input(self, state, width, grad):
        """The `state` input as the kernels take it: through the observation normalizer when one is attached (on the
        autograd graph when `grad`)."""
        x = self._input(state, width, grad)
        norm = self.obs_normalizer
        if norm is None:
            return x
        return norm.apply(x) if grad else norm.normalize(x)

    # ---- autograd path (differentiable=True) ----------------------------------------------
    def _param_list(self):
        out = []
        for name in _LAYER_NAMES:
            layer = getattr(self, name)
            out += [layer.weight, layer.bias]
        return out

    def _use_autograd(self, inputs):
        if not (self.differentiable and torch.is_grad_enabled()):
            return False
        return (any(torch.is_tensor(x) and x.requires_grad for x in inputs)
                or any(p.requires_grad for p in self._param_list()))

    def _grad_params(self):
        """The parameters as autograd inputs.  Their .grad is bound to the flat gradient buffer first, so backward
        accumulates there, where zero_grad(), SharedAdam.step() and the learner read the gradients."""
        params = self._param_list()
        if any(p.requires_grad for p in params):
            self.flat_grads()
        return params


class actor(_FlatNet):
    """models.py:15-41.  fc1 -> ReLU -> fc2 -> fc2_2 -> ReLU -> fc3 -> tanh
    (no ReLU between fc2 and fc2_2, SURVEY.md H9)."""

    @staticmethod
    def _layers(input_size, output_size):
        return [(input_size, HIDDEN), (HIDDEN, HIDDEN), (HIDDEN, HIDDEN), (HIDDEN, output_size)]

    def __init__(self, input_size, output_size, device=None, differentiable=False):
        self.input_size, self.output_size = input_size, output_size
        super().__init__(self._layers(input_size, output_size), device)
        self.differentiable = bool(differentiable)
        self.init_weights()

    @classmethod
    def unfilled(cls, input_size, output_size, device=None):
        """An actor whose flat buffer is allocated but not written: no RNG draw and no kernel.  For a buffer a kernel
        fills completely (DDPG.perturbed_actor)."""
        net = cls.__new__(cls)
        net.input_size, net.output_size = input_size, output_size
        _FlatNet.__init__(net, cls._layers(input_size, output_size), device, empty=True)
        return net

    def init_weights(self, init_w=10e-3):
        # same CPU-RNG consumption as the reference: 4 nn.Linear ctors, 3 fan-in normals, fc3 normal
        ls = [nn.Linear(i, o) for i, o in self._dims]
        _write_init(self, ls, 3e-3)

    def forward(self, state):
        _lib.require_cuda()
        if self._use_autograd((state,)):
            x = self._state_input(state, self.input_size, True)
            return _ActorFn.apply(self, int(self.precision), x, *self._grad_params())
        x = self._state_input(state, self.input_size, False)
        B = x.shape[0]
        out = torch.empty(B, self.output_size, dtype=torch.float32, device=x.device)
        _lib.check(_lib.lib().d4pg_actor_forward(_lib.ptr(self._flat), self.input_size, self.output_size,
                                                 _lib.ptr(x), B, _lib.ptr(out), _lib.ptr(self._workspace(B)),
                                                 int(self.precision), _lib.stream_ptr()), "d4pg_actor_forward")
        return out


class CriticHead(object):
    """`critic_dist_info` parsed and validated once; the critic module, DDPG and the learner read the head from here.

    kind: "categorical", "mixture_of_gaussian" or "quantile"; width: fc3's output width (N atoms, 3K, N quantiles);
    code: the learner's dist_type (0, 1, 2); n_components (K), n_quantiles (N) and kappa: None where the kind has none.
    v_min, v_max, delta and bin_centers: a categorical head's support, None elsewhere.

    learner=True parses the head as DDPG needs it for its learner: with the categorical support (a critic module has
    none), and without the range checks.  DDPG parses its head before it builds any network and the critic it builds
    makes those checks, which keeps the order in which a config's faults are reported."""

    def __init__(self, dist_info, learner=False):
        self.kind = dist_info["type"]
        self.n_components = self.n_quantiles = self.kappa = None
        self.v_min = self.v_max = self.delta = self.bin_centers = None
        if self.kind == "quantile":
            # QR-DQN: fc3 gives N quantiles at tau_k = (2k+1) / (2N); the learner's loss is the quantile-Huber loss
            # against the N bootstrapped target quantiles (csrc/qr_heads.cu); td = mean(theta) - (r + c mean(theta'))
            self.code = 2
            self.n_quantiles = self.width = int(dist_info["n_quantiles"])
            if not learner and not 2 <= self.n_quantiles <= _lib.MAX_ATOMS:
                raise _lib.D4PGError("n_quantiles must be in [2, %d], got %d" % (_lib.MAX_ATOMS, self.n_quantiles))
            self.kappa = float(dist_info.get("kappa", 1.0))
            if not learner and not (math.isfinite(self.kappa) and self.kappa > 0.0):
                raise _lib.D4PGError("kappa must be finite and > 0, got %r" % (self.kappa,))
        elif self.kind == "mixture_of_gaussian":
            # the reference stubs this branch (ddpg.py:48-50).  The learner's loss is the cross-entropy of the online
            # mixture under the target mixture, integrated with 8 Gauss-Hermite nodes per target component
            # (csrc/mog_heads.cu); td = E[Q] - (r + c E[Q'])
            self.code = 1
            self.n_components = int(dist_info["n_components"])
            if not learner and not 1 <= self.n_components <= _lib.MAX_COMPONENTS:
                raise _lib.D4PGError("n_components must be in [1, %d], got %d" % (_lib.MAX_COMPONENTS, self.n_components))
            self.width = 3 * self.n_components          # raw head: K weight logits, K means, K sigma pre-activations
        elif self.kind == "categorical":
            self.code = 0
            if learner:
                self.v_min, self.v_max, n = dist_info["v_min"], dist_info["v_max"], dist_info["n_atoms"]
                self.delta = (self.v_max - self.v_min) / float(n - 1)
                self.bin_centers = np.array([self.v_min + i * self.delta for i in range(n)]).reshape(-1, 1)
            self.width = int(dist_info["n_atoms"])
        else:
            raise NotImplementedError("critic_dist_info['type'] must be 'categorical', 'mixture_of_gaussian' or "
                                      "'quantile', got %r" % (self.kind,))


class critic(_FlatNet):
    """models.py:51-88.  fc1 -> ReLU -> cat(., action) -> fc2 -> ReLU -> fc2_2 -> ReLU -> fc3 -> softmax.

    dist_info {"type": "mixture_of_gaussian", "n_components": K} (1 <= K <= 32; the reference stubs this branch,
    models.py:63-65): fc3 is Linear(256, 3K) and forward returns (w, mu, sigma), each [B, K]: w = softmax(raw[:, :K]),
    mu = raw[:, K:2K], sigma = softplus(raw[:, 2K:]) + 1e-3.  `n_atoms` is then the raw head width 3K.

    dist_info {"type": "quantile", "n_quantiles": N, "kappa": 1.0} (2 <= N <= 128, kappa finite and > 0, default 1.0):
    fc3 is Linear(256, N), built like a categorical fc3 with N atoms, and forward returns the quantiles theta [B, N],
    the raw fc3 output (quantile k at tau_k = (2k+1) / (2N)).  `n_atoms` is N; `kappa` is the Huber threshold of the
    learner's quantile-Huber loss (it does not enter the module)."""

    def __init__(self, state_size, action_size, dist_info, device=None, differentiable=False):
        self.dist_info = dist_info
        self.head = CriticHead(dist_info)
        self.dist_type, self.n_components = self.head.kind, self.head.n_components
        self.n_quantiles, self.kappa = self.head.n_quantiles, self.head.kappa
        self.state_size, self.action_size, self.n_atoms = state_size, action_size, self.head.width
        super().__init__([(state_size, HIDDEN), (HIDDEN + action_size, HIDDEN), (HIDDEN, HIDDEN),
                          (HIDDEN, self.n_atoms)], device)
        self.differentiable = bool(differentiable)
        self.init_weights()

    def init_weights(self, init_w=10e-3):
        ls = [nn.Linear(i, o) for i, o in self._dims]
        _write_init(self, ls, 3e-4)

    def forward(self, state, action, return_logits=False):
        """Categorical: probs (and logits with return_logits).  Mixture: (w, mu, sigma) (and the raw fc3 output
        [B, 3K] as a fourth element with return_logits).  Quantile: theta [B, N], which already is the raw fc3 output
        (return_logits is ignored)."""
        _lib.require_cuda()
        grad = self._use_autograd((state, action))
        x = self._state_input(state, self.state_size, grad)
        a = self._input(action, self.action_size, grad)
        if grad:
            outs = _CriticFn.apply(self, int(self.precision), x, a, *self._grad_params())
        else:
            outs = self._head_outputs(x.shape[0], x.device, return_logits)
            self._head_forward(self._flat, x, a, outs, self._workspace(x.shape[0]), int(self.precision))
        if self.n_quantiles is not None:
            return outs[0]
        if return_logits:
            return outs
        return outs[0] if self.n_components is None else outs[:3]

    # ---- the three heads: outputs, C forward, what backward keeps, C backward ----------------------------------------
    def _head_outputs(self, B, device, raw):
        """Categorical (probs, logits), mixture (w, mu, sigma, raw), quantile (theta,).  Without `raw` the categorical
        logits and the mixture raw are None: the forward keeps them in its workspace."""
        def new(n):
            return torch.empty(B, n, dtype=torch.float32, device=device)
        if self.n_quantiles is not None:
            return (new(self.n_atoms),)
        last = new(self.n_atoms) if raw else None
        if self.n_components is not None:
            return (new(self.n_components), new(self.n_components), new(self.n_components), last)
        return (new(self.n_atoms), last)

    def _head_forward(self, flat, x, a, outs, ws, precision):
        L, P, B = _lib.lib(), _lib.ptr, x.shape[0]
        if self.n_components is not None:
            w, mu, sigma, raw = outs
            _lib.check(L.d4pg_critic_forward_mog(P(flat), self.state_size, self.action_size, self.n_components, P(x),
                                                 P(a), B, P(w), P(mu), P(sigma), P(raw), P(ws), precision,
                                                 _lib.stream_ptr()), "d4pg_critic_forward_mog")
            return
        probs, logits = (None, outs[0]) if self.n_quantiles is not None else outs
        _lib.check(L.d4pg_critic_forward(P(flat), self.state_size, self.action_size, self.n_atoms, P(x), P(a), B,
                                         P(probs), P(logits), P(ws), precision, _lib.stream_ptr()), "d4pg_critic_forward")

    def _head_saved(self, outs):
        """The outputs the head's backward reads: the categorical probs (softmax Jacobian), the mixture raw (softmax /
        softplus'); a quantile head's backward reads none."""
        if self.n_quantiles is not None:
            return ()
        return (outs[-1],) if self.n_components is not None else (outs[0],)

    def _head_backward(self, flat, x, a, saved, ws, grads, grad_flat, grad_x, grad_a, scratch, precision):
        L, P, B = _lib.lib(), _lib.ptr, x.shape[0]
        grads = [P(g) for g in grads]
        if self.n_components is not None:
            g_w, g_mu, g_sigma = grads[:3]
            _lib.check(L.d4pg_critic_backward_mog(P(flat), self.state_size, self.action_size, self.n_components, P(x),
                                                  P(a), B, P(saved[0]), P(ws), g_w, g_mu, g_sigma, P(grad_flat),
                                                  P(grad_x), P(grad_a), P(scratch), precision, _lib.stream_ptr()),
                       "d4pg_critic_backward_mog")
            return
        if self.n_quantiles is not None:        # d loss / d theta is the logits' gradient: no head Jacobian
            probs, g_probs, g_logits = None, None, grads[0]
        else:
            probs, (g_probs, g_logits) = P(saved[0]), grads
        _lib.check(L.d4pg_critic_backward(P(flat), self.state_size, self.action_size, self.n_atoms, P(x), P(a), B,
                                          probs, P(ws), g_probs, g_logits, P(grad_flat), P(grad_x), P(grad_a),
                                          P(scratch), precision, _lib.stream_ptr()), "d4pg_critic_backward")


def _backward_buffers(ctx, net, inputs, out_dim):
    """What a d4pg_*_backward call writes: the flat parameter gradient (None unless a parameter asks for one), a
    gradient for each of `inputs` (the Function's inputs from index 2) that asks for one, and the scratch -- two
    [B,256] delta planes and one output-head plane of row pitch pitch4(out_dim), at least [B,256]
    (include/d4pg_b200.h)."""
    x = inputs[0]
    want_p = any(ctx.needs_input_grad[2 + len(inputs):])
    grad_flat = torch.empty(net._total, dtype=torch.float32, device=x.device) if want_p else None
    grad_in = [torch.empty_like(t) if ctx.needs_input_grad[2 + i] else None for i, t in enumerate(inputs)]
    head = max(HIDDEN, (out_dim + 3) & ~3)
    scratch = torch.empty(x.shape[0] * (2 * HIDDEN + head), dtype=torch.float32, device=x.device)
    return grad_flat, grad_in, scratch


def _param_grads(ctx, net, grad_flat, first):
    """Per-parameter gradients as views of `grad_flat` (None where autograd did not ask), in _param_list order."""
    out = []
    for i, (w, b) in enumerate(net._views(grad_flat) if grad_flat is not None else [(None, None)] * 4):
        out += [w if ctx.needs_input_grad[first + 2 * i] else None,
                b if ctx.needs_input_grad[first + 2 * i + 1] else None]
    return out


def _f32(g):
    return g.to(dtype=torch.float32).contiguous() if g is not None else None


class _ActorFn(torch.autograd.Function):
    """action = actor(state) through d4pg_actor_forward; backward = d4pg_actor_backward.  Inputs: the module,
    the precision, the state and the 8 parameter views (so autograd routes their gradients and their version
    counters catch an in-place weight write between forward and backward)."""

    @staticmethod
    def forward(ctx, net, precision, x, *params):
        B = x.shape[0]
        out = torch.empty(B, net.output_size, dtype=torch.float32, device=x.device)
        ws = torch.empty(3 * B * HIDDEN, dtype=torch.float32, device=x.device)      # h1..h3, kept for backward
        flat = net._flat
        _lib.check(_lib.lib().d4pg_actor_forward(_lib.ptr(flat), net.input_size, net.output_size, _lib.ptr(x), B,
                                                 _lib.ptr(out), _lib.ptr(ws), precision, _lib.stream_ptr()),
                   "d4pg_actor_forward")
        ctx.net, ctx.precision, ctx.flat, ctx.ws = net, precision, flat, ws
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, out, *params)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, out = ctx.saved_tensors[:2]          # unpacking checks the version counters (parameters included)
        net = ctx.net
        if g is None:
            return (None,) * (3 + 8)
        g = _f32(g)
        grad_flat, (grad_x,), scratch = _backward_buffers(ctx, net, (x,), net.output_size)
        _lib.check(_lib.lib().d4pg_actor_backward(_lib.ptr(ctx.flat), net.input_size, net.output_size, _lib.ptr(x),
                                                  x.shape[0], _lib.ptr(out), _lib.ptr(ctx.ws), _lib.ptr(g),
                                                  _lib.ptr(grad_flat), _lib.ptr(grad_x), _lib.ptr(scratch),
                                                  ctx.precision, _lib.stream_ptr()), "d4pg_actor_backward")
        return (None, None, grad_x, *_param_grads(ctx, net, grad_flat, 3))


class _CriticFn(torch.autograd.Function):
    """critic(state, action) of any head: its outputs (critic._head_outputs, the raw one included) through the head's
    C forward; backward = the head's C backward.  A mixture's raw output is for inspection only: it is marked
    non-differentiable and its gradient is not propagated."""

    @staticmethod
    def forward(ctx, net, precision, x, a, *params):
        B = x.shape[0]
        outs = net._head_outputs(B, x.device, True)
        ws = torch.empty(3 * B * HIDDEN, dtype=torch.float32, device=x.device)      # h1..h3, kept for backward
        flat = net._flat
        net._head_forward(flat, x, a, outs, ws, precision)
        ctx.net, ctx.precision, ctx.flat, ctx.ws = net, precision, flat, ws
        ctx.set_materialize_grads(False)
        if net.n_components is not None:
            ctx.mark_non_differentiable(outs[-1])
        saved = net._head_saved(outs)
        ctx.n_saved = len(saved)
        ctx.save_for_backward(x, a, *saved, *params)
        return outs

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        x, a = ctx.saved_tensors[:2]            # unpacking checks the version counters (parameters included)
        saved = ctx.saved_tensors[2:2 + ctx.n_saved]
        net = ctx.net
        if net.n_components is not None:
            grads = grads[:3]                   # the raw output's gradient is not propagated
        if all(g is None for g in grads):
            return (None,) * (4 + 8)
        grads = [_f32(g) for g in grads]
        grad_flat, (grad_x, grad_a), scratch = _backward_buffers(ctx, net, (x, a), net.n_atoms)
        net._head_backward(ctx.flat, x, a, saved, ctx.ws, grads, grad_flat, grad_x, grad_a, scratch, ctx.precision)
        return (None, None, grad_x, grad_a, *_param_grads(ctx, net, grad_flat, 4))


def _write_init(net, cpu_linears, fc3_std):
    for l in cpu_linears[:3]:
        l.weight.data = fanin_init(l.weight.data.size())
    cpu_linears[3].weight.data.normal_(0, fc3_std)
    with torch.no_grad():
        for name, l in zip(_LAYER_NAMES, cpu_linears):
            layer = getattr(net, name)
            layer.weight.data.copy_(l.weight.data)
            layer.bias.data.copy_(l.bias.data)
