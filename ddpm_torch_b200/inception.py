"""FID Inception-v3 (``ddpm_torch/metrics/inception.py``): the TensorFlow FID network, assembled from torchvision's Inception
building blocks.  On an sm_90 device, with no gradient wanted and BatchNorm in eval mode, ``InceptionV3.forward`` runs on the
engine (``ddpm_inception_forward``: TF32 tensor-core convolutions with BatchNorm folded in, csrc/inception.cuh); everything
else (CPU, autograd, training-mode BatchNorm, ``DataParallel`` replicas, other dtypes) runs the torch modules below.
``forward(x, spatial=True)`` also returns sFID's spatial features (``spatial_features``) from the same pass, on either route.

The FID network differs from torchvision's ImageNet Inception-v3 in three places, all reproduced here:
  * 1008 classes (its ``fc`` is part of the checkpoint; only the Inception Score uses it, as ``InceptionV3.fc_weight``);
  * the 3x3 average pools inside the A, C and E blocks exclude the padding (TensorFlow's ``count_include_pad=False``);
  * the last E block (``Mixed_7c``) pools its pool branch with a 3x3 max pool.
Module names follow torchvision's ``Inception3``, so the published ``pt_inception-2015-12-05-6726825d.pth`` loads with
``strict=True``, and ``InceptionV3``'s own ``state_dict`` has the reference's ``blocks.<i>.<j>`` keys.
"""
import ctypes as C
import math
import os

import torch
import torch.nn as nn
import torch.nn.functional as F
import torchvision.models.inception as tvi

from . import _lib

FID_WEIGHTS_URL = "https://github.com/mseitzer/pytorch-fid/releases/download/fid_weights/pt_inception-2015-12-05-6726825d.pth"


def _avg3(x):
    return F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)


def _max3(x):
    return F.max_pool2d(x, kernel_size=3, stride=1, padding=1)


class _BlockA(tvi.InceptionA):
    def forward(self, x):
        b5 = self.branch5x5_2(self.branch5x5_1(x))
        b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        return torch.cat([self.branch1x1(x), b5, b3, self.branch_pool(_avg3(x))], 1)


class _BlockC(tvi.InceptionC):
    def forward(self, x):
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        d = x
        for m in (self.branch7x7dbl_1, self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4, self.branch7x7dbl_5):
            d = m(d)
        return torch.cat([self.branch1x1(x), b7, d, self.branch_pool(_avg3(x))], 1)


class _BlockE(tvi.InceptionE):
    def __init__(self, in_channels, pool):
        super().__init__(in_channels)
        self.pool = pool

    def forward(self, x):
        b3 = self.branch3x3_1(x)
        b3 = torch.cat([self.branch3x3_2a(b3), self.branch3x3_2b(b3)], 1)
        d = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        d = torch.cat([self.branch3x3dbl_3a(d), self.branch3x3dbl_3b(d)], 1)
        return torch.cat([self.branch1x1(x), b3, d, self.branch_pool(self.pool(x))], 1)


def weights_path():
    """Where the FID weights live: the torch hub checkpoint directory, as ``load_state_dict_from_url`` would keep them."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", FID_WEIGHTS_URL.rsplit("/", 1)[-1])


def fid_inception_v3():
    """torchvision's Inception3 patched into the FID network, with the FID weights loaded ``strict=True``.  The weights are
    fetched into the hub checkpoint directory only when they are not there yet."""
    net = tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False)
    net.Mixed_5b = _BlockA(192, pool_features=32)
    net.Mixed_5c = _BlockA(256, pool_features=64)
    net.Mixed_5d = _BlockA(288, pool_features=64)
    for name, c7 in (("Mixed_6b", 128), ("Mixed_6c", 160), ("Mixed_6d", 160), ("Mixed_6e", 192)):
        setattr(net, name, _BlockC(768, channels_7x7=c7))
    net.Mixed_7b = _BlockE(1280, _avg3)
    net.Mixed_7c = _BlockE(2048, _max3)
    path = weights_path()
    if not os.path.isfile(path):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        torch.hub.download_url_to_file(FID_WEIGHTS_URL, path)
    net.load_state_dict(torch.load(path, map_location="cpu"), strict=True)
    return net


class InceptionV3(nn.Module):
    """Feature maps of the FID Inception (inception.py:20-169): block 0 ends at the first max pool (64 channels), block 1 at the
    second (192), block 2 before the auxiliary classifier (768) and block 3 at the final average pool (2048).
    ``forward(x)`` returns the requested blocks' outputs in ascending order.  ``x`` is expected in [0, 1] with
    ``normalize_input`` and in [-1, 1] without; with ``resize_input`` it is first resized bilinearly to 299 x 299."""

    DEFAULT_BLOCK_INDEX = 3
    BLOCK_INDEX_BY_DIM = {64: 0, 192: 1, 768: 2, 2048: 3}

    def __init__(self, output_blocks=(DEFAULT_BLOCK_INDEX,), resize_input=True, normalize_input=False, requires_grad=False,
                 use_fid_inception=True):
        super().__init__()
        if not use_fid_inception:
            raise ValueError("only the FID Inception (use_fid_inception=True) is provided")
        self.resize_input = resize_input
        self.normalize_input = normalize_input
        self.output_blocks = sorted(output_blocks)
        self.last_needed_block = max(output_blocks)
        assert self.last_needed_block <= 3, "Last possible output block index is 3"
        net = fid_inception_v3()
        stages = [
            [net.Conv2d_1a_3x3, net.Conv2d_2a_3x3, net.Conv2d_2b_3x3, nn.MaxPool2d(kernel_size=3, stride=2)],
            [net.Conv2d_3b_1x1, net.Conv2d_4a_3x3, nn.MaxPool2d(kernel_size=3, stride=2)],
            [net.Mixed_5b, net.Mixed_5c, net.Mixed_5d, net.Mixed_6a, net.Mixed_6b, net.Mixed_6c, net.Mixed_6d, net.Mixed_6e],
            [net.Mixed_7a, net.Mixed_7b, net.Mixed_7c, nn.AdaptiveAvgPool2d(output_size=(1, 1))],
        ]
        self.blocks = nn.ModuleList(nn.Sequential(*s) for s in stages[:self.last_needed_block + 1])
        # the checkpoint's 1008-way fc weight [1008, 2048] (the Inception Score's logits, metrics.InceptionScore): a plain CPU
        # tensor, so it is neither in the state_dict nor moved or replicated with the module
        self.fc_weight = net.fc.weight.detach()
        self.requires_grad_(requires_grad)
        self.use_engine = True             # False: always the torch modules (InceptionStatistics over a device list)
        self._native_tensors = None        # the engine's raw parameters, in its order (None: not gathered yet)
        self._packed = None
        self._packed_key = None
        self._ws = None
        self._load_epoch = 0
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._weights_changed())

    def _weights_changed(self):
        self._load_epoch += 1
        self._packed_key = None

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)      # .to() / .cuda() may give buffers new tensors
        self._native_tensors = None
        self._packed_key = None
        return out

    def _engine_tensors(self):
        """The module's conv weights and BatchNorm vectors in the engine's parameter order (ddpm_inception_param_info), or
        None for the entries of blocks this module does not hold."""
        if self._native_tensors is None:
            own = dict(self.named_parameters())
            own.update(self.named_buffers())
            L = _lib.lib()
            out = []
            for i in range(L.ddpm_inception_num_params()):
                name, ndim, dims, off = C.c_char_p(), C.c_int(), (C.c_int * 4)(), C.c_longlong()
                _lib.check(L.ddpm_inception_param_info(i, C.byref(name), C.byref(ndim), C.byref(dims), C.byref(off)), "inception_param_info")
                mod, rest = name.value.decode().split(".", 1)
                key = f"{_ENGINE_BLOCK[mod]}.{rest}"
                shape = tuple(dims[:ndim.value])
                out.append((own.get(key), shape, off.value))
            self._native_tensors = out
        return self._native_tensors

    def native_eligible(self, inp):
        """True when ``forward(inp)`` runs on the engine: every parameter on one sm_90 CUDA device in fp32, BatchNorm in eval
        mode, no gradient wanted, ``use_engine`` set, and ``inp`` a non-empty 4-D CUDA fp32 batch of 3-channel images on that
        device.  ``DataParallel`` replicas always take the torch path."""
        if not self.use_engine or getattr(self, "_is_replica", False) or not isinstance(inp, torch.Tensor):
            return False
        if not (inp.is_cuda and inp.dim() == 4 and inp.shape[0] > 0 and inp.shape[1] == 3 and inp.dtype == torch.float32):
            return False
        if torch.is_grad_enabled() and (inp.requires_grad or any(p.requires_grad for p in self.parameters())):
            return False
        if any(m.training for m in self.modules()):
            return False
        ts = [t for t, _, _ in self._engine_tensors() if t is not None]
        if any(t.device != inp.device or t.dtype != torch.float32 for t in ts):
            return False
        return torch.cuda.get_device_capability(inp.device) == (9, 0)

    def _repack_if_needed(self, dev):
        ents = [t for t, _, _ in self._engine_tensors() if t is not None]
        if any(t.is_inference() for t in ents):
            key = None                         # inference tensors keep no version counter: pack on every call
        else:
            key = (dev, self._load_epoch, sum(t._version for t in ents), sum(t.data_ptr() for t in ents))
        if key is not None and key == self._packed_key:
            return
        ents = self._engine_tensors()
        L = _lib.lib()
        parts = [t.detach().reshape(-1) if t is not None else torch.zeros(math.prod(shape), dtype=torch.float32, device=dev) for t, shape, _ in ents]
        raw = torch.cat(parts)
        if self._packed is None or self._packed.device != dev:
            self._packed = torch.empty(L.ddpm_inception_packed_bytes(), dtype=torch.uint8, device=dev)
        _lib.check(L.ddpm_inception_pack(raw.data_ptr(), self._packed.data_ptr(), _lib.stream_ptr(dev)), "inception_pack")
        self._packed_key = key

    def forward_native(self, inp, pooled=False, spatial=False):
        """The engine's forward of ``inp`` (see ``native_eligible``): the requested blocks' outputs, NCHW fp32 as ``forward``
        returns them; with ``pooled`` instead the [N, C] global average of the last needed block (InceptionStatistics).  With
        ``spatial`` the return value is a pair: that result and sFID's [N, 7 h w] features (``spatial_features``), gathered by
        the engine from Mixed_6d's output in the same pass."""
        dev = inp.device
        L = _lib.lib()
        self._check_spatial(spatial)
        with torch.cuda.device(dev):
            self._repack_if_needed(dev)
            x = inp.contiguous()
            N, _, H, W = x.shape
            last = self.last_needed_block
            need = L.ddpm_inception_workspace_bytes(N, H, W, int(self.resize_input), last)
            if need < 0:
                _lib.check(int(need), "InceptionV3")
            if self._ws is None or self._ws.device != dev or self._ws.numel() < need:
                self._ws = None
                self._ws = torch.empty(int(need), dtype=torch.uint8, device=dev)
            outs = (C.c_void_p * 4)()
            res = []
            feats = None
            if pooled:
                feats = torch.empty(N, _BLOCK_CHANNELS[last], dtype=torch.float32, device=dev)
            else:
                for b in self.output_blocks:
                    h, w = _block_hw(H, W, self.resize_input, b)
                    res.append(torch.empty(N, _BLOCK_CHANNELS[b], h, w, dtype=torch.float32, device=dev))
                    outs[b] = res[-1].data_ptr()
            sp = None
            if spatial:
                h, w = _block_hw(H, W, self.resize_input, 2)
                sp = torch.empty(N, h * w * SPATIAL_CHANNELS, dtype=torch.float32, device=dev)
            _lib.check(L.ddpm_inception_forward_ex(self._packed.data_ptr(), x.data_ptr(), N, H, W, int(self.resize_input),
                                                   int(self.normalize_input), last, C.byref(outs),
                                                   None if feats is None else feats.data_ptr(),
                                                   None if sp is None else sp.data_ptr(), self._ws.data_ptr(), self._ws.numel(),
                                                   _lib.stream_ptr(dev)), "InceptionV3")
        out = feats if pooled else res
        return (out, sp) if spatial else out

    def _check_spatial(self, spatial):
        if spatial and self.last_needed_block < 2:
            raise ValueError("spatial features come from Mixed_6d, in block 2; this module stops at block "
                             f"{self.last_needed_block}")

    def forward(self, inp, spatial=False):
        """The requested blocks' outputs; with ``spatial`` a pair of those and sFID's [N, 7 h w] features
        (``spatial_features`` of Mixed_6d's output), from the same pass."""
        self._check_spatial(spatial)
        if self.native_eligible(inp):
            return self.forward_native(inp, spatial=spatial)
        x = inp
        if self.resize_input:
            x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
        if self.normalize_input:
            x = 2 * x - 1
        out, sp = [], None
        for i, block in enumerate(self.blocks):
            if spatial and i == 2:
                # module by module rather than through a hook, so that DataParallel replicas return the features too
                for j, m in enumerate(block):
                    x = m(x)
                    if j == _MIXED_6D:
                        sp = spatial_features(x)
            else:
                x = block(x)
            if i in self.output_blocks:
                out.append(x)
        return (out, sp) if spatial else out


def spatial_features(mixed_6d):
    """sFID's spatial features (Nash et al., 2021) from Mixed_6d's NCHW output [N, 768, h, w]: channels [0, 7), which are
    its branch1x1 after BatchNorm and ReLU (the first slice of the block's torch.cat), flattened in TensorFlow's NHWC order,
    feature (y w + x) 7 + c: [N, 7 h w], 2023 features at 299 x 299.

    This follows the guided-diffusion evaluator (Dhariwal & Nichol, 2021), which reads ``mixed_6/conv:0[..., :7]`` from the
    TensorFlow 2015 Inception graph.  That ``mixed_6`` is ``Mixed_6d`` (``mixed_3`` is ``Mixed_6a``; ``mixed_4``..``mixed_7``
    are ``6b``..``6e``) and that ``mixed_6/conv:0`` is the post-ReLU output of its 1x1 branch is assumed, not verified: the
    values are meant to be comparable to ADM's sFID but have not been checked against it."""
    return mixed_6d[:, :SPATIAL_CHANNELS].permute(0, 2, 3, 1).reshape(mixed_6d.shape[0], -1)


_ENGINE_BLOCK = {"Conv2d_1a_3x3": "blocks.0.0", "Conv2d_2a_3x3": "blocks.0.1", "Conv2d_2b_3x3": "blocks.0.2",
                 "Conv2d_3b_1x1": "blocks.1.0", "Conv2d_4a_3x3": "blocks.1.1",
                 **{f"Mixed_{m}": f"blocks.2.{i}" for i, m in enumerate(("5b", "5c", "5d", "6a", "6b", "6c", "6d", "6e"))},
                 **{f"Mixed_{m}": f"blocks.3.{i}" for i, m in enumerate(("7a", "7b", "7c"))}}
_BLOCK_CHANNELS = (64, 192, 768, 2048)
_MIXED_6D = 6                                    # its position in block 2
SPATIAL_CHANNELS = 7                             # sFID keeps channels [0, 7) of Mixed_6d


def _block_hw(H, W, resize, block):
    """Spatial size of block ``block``'s output for an H x W input."""
    def one(n):
        n = 299 if resize else n
        n = (n - 3) // 2 + 1 - 2                  # Conv2d_1a (3x3 s2), Conv2d_2a (3x3); Conv2d_2b keeps the size
        n = (n - 3) // 2 + 1                      # max pool: block 0
        if block >= 1:
            n = (n - 2 - 3) // 2 + 1              # Conv2d_4a (3x3), max pool: block 1
        if block >= 2:
            n = (n - 3) // 2 + 1                  # Mixed_6a: block 2
        return 1 if block == 3 else n
    return one(H), one(W)


def seeded_state_dict(seed=0):
    """A deterministic stand-in for the FID weights, for tests and benchmarks that must not reach the network: every
    floating entry of the FID network's state dict drawn from ``torch.Generator().manual_seed(seed)`` in key order --
    convolution / fc weights N(0, 2 / fan_in), BatchNorm weights 1 + 0.1 N(0, 1), biases and running means 0.1 N(0, 1),
    running variances U(0.5, 1.5) (positive) -- and ``num_batches_tracked`` = 0."""
    net = tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False)
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in net.state_dict().items():
        if k.endswith("num_batches_tracked"):
            out[k] = torch.zeros_like(v)
        elif k.endswith("running_var"):
            out[k] = torch.rand(v.shape, generator=g) + 0.5
        elif k.endswith("bn.weight"):
            out[k] = 1 + 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith("weight"):
            out[k] = torch.randn(v.shape, generator=g) * (2.0 / v[0].numel()) ** 0.5
        else:                                   # biases, running means
            out[k] = 0.1 * torch.randn(v.shape, generator=g)
    return out
