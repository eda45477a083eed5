"""``Decoder`` of ddpm_torch/toy/toy_model.py on the toy engine (csrc/toy_mlp.cuh).

The module tree, parameter creation order and initialisation are the reference's, so the same seed gives bit-identical weights
and reference checkpoints load with ``strict=True``.  ``temp_fc`` repeats ONE ``TemporalLayer`` (``[layer] * n``, as upstream):
its 8 parameters appear under every index of ``state_dict()`` (31 keys for 3 layers) and once in ``parameters()`` (15).

Parameters are ordinary fp32 tensors: any optimiser updates them in place, and every engine call passes their current pointers,
so there is no packed copy to refresh.  A CUDA model runs its forward and backward on the engine; a CPU model raises."""
import ctypes as C
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib


class Linear(nn.Module):
    """modules.py:37-66: xavier_uniform weight, zero bias."""

    def __init__(self, in_features, out_features, bias=True, init_scale=1.):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty((out_features, in_features), dtype=torch.float32))
        if bias:
            self.bias = nn.Parameter(torch.empty((out_features,), dtype=torch.float32))
        else:
            self.register_parameter("bias", None)
        self.init_scale = init_scale
        nn.init.xavier_uniform_(self.weight, gain=math.sqrt(init_scale or 1e-10))
        if self.bias is not None:
            nn.init.zeros_(self.bias)

    def forward(self, x):
        return F.linear(x, self.weight, self.bias)

    def extra_repr(self):
        return f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}"


class Sequential(nn.Sequential):
    pass


class TemporalLayer(nn.Module):
    def __init__(self, in_features, out_features, temporal_features):
        super().__init__()
        self.norm1 = nn.LayerNorm(in_features)
        self.fc1 = Linear(in_features, out_features, bias=False)
        self.norm2 = nn.LayerNorm(out_features)
        self.fc2 = Linear(out_features, out_features, bias=False)
        self.enc = Linear(temporal_features, out_features)
        self.skip = nn.Identity()


class ToyCfg(C.Structure):
    _fields_ = [("in_features", C.c_int), ("mid_features", C.c_int), ("num_layers", C.c_int)]


class ToyParams(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "in_fc_weight", "norm1_weight", "norm1_bias", "fc1_weight", "norm2_weight", "norm2_bias", "fc2_weight", "enc_weight",
        "enc_bias", "out_norm_weight", "out_norm_bias", "out_fc_weight", "out_fc_bias", "t_proj_weight", "t_proj_bias")]


class Decoder(nn.Module):
    def __init__(self, in_features, mid_features, num_temporal_layers):
        super().__init__()
        self.in_fc = Linear(in_features, mid_features, bias=False)
        self.temp_fc = Sequential(*([TemporalLayer(mid_features, mid_features, mid_features)] * num_temporal_layers))
        self.out_norm = nn.LayerNorm(mid_features)
        self.out_fc = Linear(mid_features, in_features)
        self.t_proj = nn.Sequential(Linear(mid_features, mid_features), nn.LeakyReLU(negative_slope=0.02, inplace=True))
        self.in_features, self.mid_features, self.num_temporal_layers = in_features, mid_features, num_temporal_layers

    # ------------------------------------------------------------------ engine plumbing
    def _cfg(self):
        return ToyCfg(self.in_features, self.mid_features, self.num_temporal_layers)

    def _param_table(self):
        ps = list(self.parameters())
        return ToyParams(*[p.data_ptr() for p in ps])

    def _check(self, x):
        dev = self.in_fc.weight.device
        if dev.type != "cuda":
            raise RuntimeError("ddpm_torch_b200.toy.Decoder runs on the toy engine only: move the model to a CUDA device")
        if x.device != dev:
            raise RuntimeError(f"Decoder lives on {dev} but the input is on {x.device}")
        if any(p.dtype != torch.float32 or not p.is_contiguous() for p in self.parameters()):
            raise RuntimeError("Decoder parameters must be contiguous fp32 tensors")
        return dev

    def _workspace(self, rows, training, dev):
        n = _lib.lib().ddpm_toy_workspace_bytes(C.byref(self._cfg()), rows, int(training))
        if n < 0:
            _lib.check(n, "toy_workspace_bytes")
        return torch.empty(max(int(n), 256), dtype=torch.uint8, device=dev)

    def forward(self, x, t):
        dev = self._check(x)
        t = torch.as_tensor(t, device=dev).to(torch.int64).reshape(-1).contiguous()
        # decided here: inside the autograd Function's forward, grad mode is always off
        train = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters()))
        return _DecoderFn.apply(self, train, x.contiguous().float(), t, *self.parameters())


class _DecoderFn(torch.autograd.Function):
    """out = Decoder(x, t) through ddpm_toy_forward / ddpm_toy_backward, with gradients for x and every parameter."""

    @staticmethod
    def forward(ctx, model, train, x, t, *params):
        B = x.shape[0]
        if x.ndim != 2 or x.shape[1] != model.in_features or t.numel() != B:
            raise ValueError(f"Decoder expects x [B, {model.in_features}] and t [B], got {list(x.shape)} and {list(t.shape)}")
        dev = x.device
        out = torch.empty_like(x)
        ws = model._workspace(B, train, dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ddpm_toy_forward(C.byref(model._cfg()), C.byref(model._param_table()), x.data_ptr(), t.data_ptr(), B,
                                                   out.data_ptr(), int(train), ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)),
                       "toy_forward")
        ctx.model, ctx.ws, ctx.t, ctx.x_grad = model, ws, t, x.requires_grad
        return out

    @staticmethod
    def backward(ctx, d_out):
        model = ctx.model
        d_out = d_out.contiguous().float()
        B = d_out.shape[0]
        dev = d_out.device
        flat = torch.empty(sum(p.numel() for p in model.parameters()), dtype=torch.float32, device=dev)
        dx = torch.empty_like(d_out) if ctx.x_grad else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ddpm_toy_backward(C.byref(model._cfg()), C.byref(model._param_table()), ctx.t.data_ptr(), d_out.data_ptr(),
                                                    B, dx.data_ptr() if dx is not None else None, flat.data_ptr(), ctx.ws.data_ptr(),
                                                    ctx.ws.numel(), _lib.stream_ptr(dev)), "toy_backward")
        return (None, None, dx, None, *_split(flat, model))


def _split(flat, model):
    out, o = [], 0
    for p in model.parameters():
        out.append(flat[o:o + p.numel()].view_as(p))
        o += p.numel()
    return out
