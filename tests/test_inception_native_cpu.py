"""The engine's FID Inception-v3 forward without a GPU: the parameter inventory and layer table against the torch module, the
workspace sizes, argument refusals, exports, the convolution kernel's SASS and the BatchNorm fold.  Nothing reaches the network."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import inception as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "ddpm_torch_b200", "libddpm_b200.so")
NAMES = ("ddpm_inception_num_params", "ddpm_inception_param_info", "ddpm_inception_conv_info", "ddpm_inception_packed_bytes",
         "ddpm_inception_pack", "ddpm_inception_workspace_bytes", "ddpm_inception_forward", "ddpm_inception_conv_scratch_bytes",
         "ddpm_inception_conv_run", "ddpm_inception_pool_run", "ddpm_inception_input_run")


@pytest.fixture
def offline(monkeypatch, tmp_path):
    def refuse(*a, **k):
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    os.makedirs(os.path.dirname(I.weights_path()))
    torch.save(I.seeded_state_dict(0), I.weights_path())


def inventory():
    L = _lib.lib()
    out = []
    for i in range(L.ddpm_inception_num_params()):
        name, nd, dims, off = C.c_char_p(), C.c_int(), (C.c_int * 4)(), C.c_longlong()
        assert L.ddpm_inception_param_info(i, C.byref(name), C.byref(nd), C.byref(dims), C.byref(off)) == 0
        out.append((name.value.decode(), tuple(dims[:nd.value]), off.value))
    return out


def conv_info(i):
    info = (C.c_int * 11)()
    assert _lib.lib().ddpm_inception_conv_info(i, C.byref(info)) == 0
    return list(info)


def test_inventory_is_the_state_dict(offline):
    sd = I.fid_inception_v3().state_dict()
    want = [(k, tuple(v.shape)) for k, v in sd.items() if not k.endswith("num_batches_tracked") and not k.startswith("fc.")]
    inv = inventory()
    assert [(n, s) for n, s, _ in inv] == want
    off = 0
    for _, s, o in inv:                                     # one flat buffer, in key order, no gaps
        assert o == off
        off += int(torch.Size(s).numel())
    # the module's own names map onto every entry
    net = I.InceptionV3([0, 1, 2, 3])
    ents = net._engine_tensors()
    assert len(ents) == len(inv) and all(t is not None and tuple(t.shape) == s for t, s, _ in ents)


def test_layer_table_order_shapes_and_concat_offsets(offline):
    """Every conv once, in the order the torch forward calls them, with its kernel, stride and padding; each conv that ends a
    branch writes the channels its output occupies in the block's torch.cat."""
    net = I.InceptionV3([0, 1, 2, 3]).eval()
    calls, outs = [], {}
    convs = [(n, m) for n, m in net.named_modules() if isinstance(m, torch.nn.Conv2d)]
    def record(n):
        def hook(m, i, o):
            calls.append(n)
            outs[n] = o
        return hook
    hooks = [m.register_forward_hook(record(n)) for n, m in convs]
    block_outs = {}
    mixed = [(n, m) for n, m in net.named_modules() if n.count(".") == 2 and n.startswith("blocks.")]
    def keep(n):
        def hook(m, i, o):
            block_outs[n] = o
        return hook
    hooks += [m.register_forward_hook(keep(n)) for n, m in mixed]
    with torch.inference_mode():
        net(torch.rand(1, 3, 32, 32, generator=torch.Generator().manual_seed(0)))
    for h in hooks:
        h.remove()
    assert len(calls) == 94 and len(set(calls)) == 94
    inv = inventory()
    mods = dict(net.named_modules())
    table = {inv[5 * i][0][: -len(".conv.weight")]: i for i in range(94)}
    infos = [conv_info(i) for i in range(94)]
    assert sorted(f[10] for f in infos) == list(range(94))          # every conv once
    for step, call in enumerate(calls):
        prefix = call[: -len(".conv")]
        i = table[_tv_name(prefix)]
        cin, cout, kh, kw, st, ph, pw, c_off, c_total, to_trunk, at = infos[i]
        assert at == step                                            # in the order the torch forward runs them
        mod = mods[call]
        assert (cin, cout, (kh, kw), st, (ph, pw)) == (mod.in_channels, mod.out_channels, mod.kernel_size, mod.stride[0], mod.padding)
        if prefix.count(".") == 2:                        # stem: a whole tensor of the trunk
            assert to_trunk and (c_off, c_total) == (0, cout)
        elif to_trunk:                                    # a branch's last conv: its slice of the block's torch.cat
            blk = prefix.rsplit(".", 1)[0]
            with torch.inference_mode():
                y = F.relu(mods[prefix].bn(outs[call]))
            assert c_total == block_outs[blk].shape[1]
            assert torch.equal(block_outs[blk][:, c_off:c_off + cout], y)
        else:                                             # an intermediate of a branch
            assert (c_off, c_total) == (0, cout)
    # 5 stem convs; branch ends: 4 per A block, 2 in Mixed_6a, 4 per C block, 2 in Mixed_7a, 6 per E block
    assert sum(conv_info(i)[9] for i in range(94)) == 5 + 3 * 4 + 2 + 4 * 4 + 2 + 2 * 6


def _tv_name(prefix):
    rev = {v: k for k, v in I._ENGINE_BLOCK.items()}
    parts = prefix.split(".")
    head = ".".join(parts[:3])
    return ".".join([rev[head]] + parts[3:])


@pytest.mark.parametrize("N", [1, 3, 512])
@pytest.mark.parametrize("size", [32, 64, 256, 299])
def test_workspace_sizes(N, size):
    L = _lib.lib()
    for resize in (0, 1):
        Hi = 299 if resize else size
        for blk in range(4):
            got = L.ddpm_inception_workspace_bytes(N, size, size, resize, blk)
            h = I._block_hw(size, size, resize, min(blk, 2))[0]
            if h < 1 or (blk == 3 and (h - 3) // 2 + 1 < 1):
                assert got < 0 and b"too small" in L.ddpm_last_error()
                continue
            assert got > 0
            h1 = (Hi - 3) // 2 + 1
            # at least the split input image and the trunk buffers holding Conv2d_2a's and Conv2d_2b's outputs; at most that image
            # and five buffers of Conv2d_1a's output size at 64 channels (no later tensor is larger per image)
            assert got >= 4 * N * (Hi * Hi * 12 + (h1 - 2) ** 2 * (32 + 64))
            assert got <= 4 * N * (Hi * Hi * 12 + 5 * h1 * h1 * 64) + 6 * 256
            one = L.ddpm_inception_workspace_bytes(1, size, size, resize, blk)
            assert abs(got - N * one) <= 6 * 256 * N                   # per-image sizes, each buffer 256-byte aligned


def test_refusals():
    L = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = C.addressof(buf) + (-C.addressof(buf)) % 256
    outs = (C.c_void_p * 4)()
    assert L.ddpm_inception_workspace_bytes(0, 32, 32, 1, 3) < 0
    assert L.ddpm_inception_workspace_bytes(1, 32, 32, 2, 3) < 0
    assert L.ddpm_inception_workspace_bytes(1, 32, 32, 1, 4) < 0
    assert L.ddpm_inception_workspace_bytes(1, 32, 32, 0, 3) < 0          # too small without the resize
    fwd = L.ddpm_inception_forward
    assert fwd(None, p, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p, 1 << 40, None) < 0          # null packed
    assert fwd(p + 16, p, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p, 1 << 40, None) < 0        # misaligned packed
    assert fwd(p, None, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p, 1 << 40, None) < 0          # null x
    assert fwd(p, p, 1, 32, 32, 1, 2, 3, C.byref(outs), None, p, 1 << 40, None) < 0            # normalize
    assert fwd(p, p, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p, 16, None) < 0                  # workspace too small
    assert fwd(p, p, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p + 8, 1 << 40, None) < 0        # misaligned workspace
    bad = (C.c_void_p * 4)(None, None, None, p)
    assert fwd(p, p, 1, 32, 32, 1, 0, 2, C.byref(bad), None, p, 1 << 40, None) < 0             # output of a block not run
    assert b"outs[3]" in L.ddpm_last_error()
    assert L.ddpm_inception_pack(None, p, None) < 0 and L.ddpm_inception_pack(p, p + 4, None) < 0
    assert L.ddpm_inception_param_info(470, None, None, None, None) < 0 and L.ddpm_inception_param_info(-1, None, None, None, None) < 0
    assert L.ddpm_inception_conv_info(94, (C.c_int * 11)()) < 0
    d = _lib.IncConvDesc(N=1, H=8, W=8, Cin=32, Cout=64, kh=3, kw=3, stride=1, ph=1, pw=1, c_off=0, C_total=64)
    assert L.ddpm_inception_conv_scratch_bytes(C.byref(d)) > 0
    for field, v in (("Cout", 63), ("kh", 8), ("stride", 3), ("ph", 3), ("c_off", 2), ("C_total", 63), ("N", 0)):
        e = _lib.IncConvDesc.from_buffer_copy(d)
        setattr(e, field, v)
        assert L.ddpm_inception_conv_scratch_bytes(C.byref(e)) < 0, field
    d.scratch_bytes = 1 << 30
    d.x = d.w = d.gamma = d.beta = d.mean = d.var = d.out = d.scratch = p
    d.x = p + 4
    assert L.ddpm_inception_conv_run(C.byref(d), None) < 0                                     # x not 16-byte aligned
    d.x = p
    d.scratch_bytes = 16
    assert L.ddpm_inception_conv_run(C.byref(d), None) < 0                                     # scratch too small
    assert L.ddpm_inception_pool_run(3, p, 1, 8, 8, 4, p, 0, 4, None) < 0
    assert L.ddpm_inception_pool_run(0, p, 1, 2, 8, 4, p, 0, 4, None) < 0                      # empty output
    assert L.ddpm_inception_pool_run(1, p, 1, 8, 8, 4, p, 2, 4, None) < 0                      # slice outside C_total
    assert L.ddpm_inception_input_run(p, 1, 8, 8, 1, 0, p + 4, None) < 0


def test_exports():
    hdr = open(os.path.join(ROOT, "include", "ddpm_b200.h")).read()
    for name in NAMES:
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)
        assert re.search(r"\b" + name + r"\(", hdr)


def test_conv_kernel_sass_and_spills():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    per, cur = {}, None
    for ln in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1); per[cur] = set(); continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", ln)
        if m and cur:
            per[cur].add(m.group(1))
    convs = {fn: ops for fn, ops in per.items() if "inc_conv_tf32_kernel" in fn}
    assert len(convs) == 2
    for ops in convs.values():
        assert any(o.startswith("HGMMA") for o in ops)
        assert not any(o.startswith(("HMMA", "IMMA")) for o in ops)
    others = {fn: ops for fn, ops in per.items() if "k_inc_" in fn}
    assert len(others) == 5 and not any(o.startswith(("HGMMA", "HMMA", "IMMA")) for ops in others.values() for o in ops)
    log = os.path.join(ROOT, "ddpm_torch_b200", "csrc", "build.log")
    if not os.path.exists(log):
        pytest.skip("no build log (-Xptxas -v) next to the sources")
    lines = open(log).read().splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and ("inc_conv_tf32_kernel" in ln or "k_inc_" in ln):
            seen += 1
            spill = next(x for x in lines[i + 1:i + 5] if "bytes spill stores" in x)
            assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", spill), (ln, spill)
    assert seen == 7


def test_bn_fold_in_fp64_matches_basicconv2d_eval():
    import torchvision.models.inception as tvi
    g = torch.Generator().manual_seed(1)
    for cin, cout, k, pad in ((32, 64, (3, 3), (1, 1)), (160, 160, (1, 7), (0, 3)), (3, 32, (3, 3), (0, 0))):
        m = tvi.BasicConv2d(cin, cout, kernel_size=k, padding=pad).eval()
        with torch.no_grad():
            m.conv.weight.copy_(torch.randn(m.conv.weight.shape, generator=g) * (2 / (cin * k[0] * k[1])) ** 0.5)
            m.bn.weight.copy_(1 + 0.1 * torch.randn(cout, generator=g))
            m.bn.bias.copy_(0.1 * torch.randn(cout, generator=g))
            m.bn.running_mean.copy_(0.1 * torch.randn(cout, generator=g))
            m.bn.running_var.copy_(torch.rand(cout, generator=g) + 0.5)
        x = torch.randn(2, cin, 9, 11, generator=g)
        s = m.bn.weight.double() / torch.sqrt(m.bn.running_var.double() + 1e-3)
        wf = (m.conv.weight.double() * s[:, None, None, None]).float()
        bf = (m.bn.bias.double() - m.bn.running_mean.double() * s).float()
        y = F.relu(F.conv2d(x.double(), wf.double(), bf.double(), padding=pad))
        with torch.no_grad():
            want = m(x).double()
            z = F.conv2d(x.double(), m.conv.weight.double(), None, padding=pad)
            S = F.conv2d(x.double().abs(), m.conv.weight.double().abs(), None, padding=pad)
        # fp32 rounding of the torch module (conv over K terms, then the BatchNorm affine) and of the two folded values
        K = cin * k[0] * k[1]
        eps = 2.0 ** -24
        scale = s.abs()[None, :, None, None]
        bound = (K + 4) * eps * S * scale + 4 * eps * (z.abs() * scale + m.bn.bias.double().abs()[None, :, None, None]
                                                       + (m.bn.running_mean.double() * s).abs()[None, :, None, None])
        assert torch.all((y - want).abs() <= bound)
