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
import numpy as np
import torch
import torch.nn as nn

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

    def __init__(self, dims, device=None):
        super().__init__()
        self._dims = list(dims)
        self._offsets, self._sizes, self._total, self._pitch = _layout_py(self._dims)
        self._device = torch.device(device) if device is not None else default_device()
        self._flat = torch.zeros(self._total, dtype=torch.float32, device=self._device)
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
        """Flat gradient buffer (allocated on first use); `.grad` of every parameter views it."""
        if self._flat_grad is None:
            self._flat_grad = torch.zeros_like(self._flat)
            self._bind_grads()
        return self._flat_grad

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

    def share_memory(self):
        # CUDA storage is already visible to every stream of the process; the reference's
        # cross-process sharing (ddpg.py:96-98) is replaced by NCCL data parallelism.
        return self

    def zero_grad(self, set_to_none=False):
        if self._flat_grad is not None:
            self._flat_grad.zero_()

    def _workspace(self, B):
        need = 3 * B * HIDDEN
        ws = getattr(self, "_ws", None)
        if ws is None or ws.numel() < need or ws.device != self._flat.device:
            ws = torch.empty(need, dtype=torch.float32, device=self._flat.device)
            self._ws = ws
        return ws

    def _as_input(self, x, width):
        if not torch.is_tensor(x):
            x = torch.as_tensor(np.asarray(x))
        x = x.detach().to(device=self._flat.device, dtype=torch.float32)
        if x.dim() == 1:
            x = x.view(1, -1)
        assert x.shape[1] == width, "expected input width %d, got %s" % (width, tuple(x.shape))
        return x.contiguous()


class actor(_FlatNet):
    """models.py:15-41.  fc1 -> ReLU -> fc2 -> fc2_2 -> ReLU -> fc3 -> tanh
    (no ReLU between fc2 and fc2_2, SURVEY.md H9)."""

    def __init__(self, input_size, output_size, device=None):
        self.input_size, self.output_size = input_size, output_size
        super().__init__([(input_size, HIDDEN), (HIDDEN, HIDDEN), (HIDDEN, HIDDEN), (HIDDEN, output_size)], device)
        self.init_weights()

    def init_weights(self, init_w=10e-3):
        # same CPU-RNG consumption as the reference: 4 nn.Linear ctors, 3 fan-in normals, fc3 normal
        ls = [nn.Linear(i, o) for i, o in self._dims]
        _write_init(self, ls, 3e-3)

    def forward(self, state):
        _lib.require_cuda()
        x = self._as_input(state, self.input_size)
        B = x.shape[0]
        out = torch.empty(B, self.output_size, dtype=torch.float32, device=x.device)
        _lib.check(_lib.lib().d4pg_actor_forward(_lib.ptr(self._flat), self.input_size, self.output_size,
                                                 _lib.ptr(x), B, _lib.ptr(out), _lib.ptr(self._workspace(B)),
                                                 int(self.precision), _lib.stream_ptr()), "d4pg_actor_forward")
        return out


class critic(_FlatNet):
    """models.py:51-88.  fc1 -> ReLU -> cat(., action) -> fc2 -> ReLU -> fc2_2 -> ReLU -> fc3 -> softmax."""

    def __init__(self, state_size, action_size, dist_info, device=None):
        self.dist_info = dist_info
        if dist_info["type"] != "categorical":
            raise NotImplementedError("only the categorical head exists (mixture_of_gaussian is a TODO stub "
                                      "in the reference too, models.py:63-65)")
        self.state_size, self.action_size, self.n_atoms = state_size, action_size, int(dist_info["n_atoms"])
        super().__init__([(state_size, HIDDEN), (HIDDEN + action_size, HIDDEN), (HIDDEN, HIDDEN),
                          (HIDDEN, self.n_atoms)], device)
        self.init_weights()

    def init_weights(self, init_w=10e-3):
        ls = [nn.Linear(i, o) for i, o in self._dims]
        _write_init(self, ls, 3e-4)

    def forward(self, state, action, return_logits=False):
        _lib.require_cuda()
        x = self._as_input(state, self.state_size)
        a = self._as_input(action, self.action_size)
        B = x.shape[0]
        probs = torch.empty(B, self.n_atoms, dtype=torch.float32, device=x.device)
        logits = torch.empty_like(probs) if return_logits else None
        _lib.check(_lib.lib().d4pg_critic_forward(_lib.ptr(self._flat), self.state_size, self.action_size, self.n_atoms,
                                                  _lib.ptr(x), _lib.ptr(a), B, _lib.ptr(probs), _lib.ptr(logits),
                                                  _lib.ptr(self._workspace(B)), int(self.precision), _lib.stream_ptr()),
                   "d4pg_critic_forward")
        return (probs, logits) if return_logits else probs


def _write_init(net, cpu_linears, fc3_std):
    for l in cpu_linears[:3]:
        l.weight.data = fanin_init(l.weight.data.size())
    cpu_linears[3].weight.data.normal_(0, fc3_std)
    with torch.no_grad():
        for name, l in zip(_LAYER_NAMES, cpu_linears):
            layer = getattr(net, name)
            layer.weight.data.copy_(l.weight.data)
            layer.bias.data.copy_(l.bias.data)
