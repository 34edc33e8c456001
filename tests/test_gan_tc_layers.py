"""GPU tests of the tensor-core (wgmma) tap-conv kernel, one layer at a time (mb_gan_debug_layer).

Reference for each layer = torch-CPU conv on operands rounded to fp16 exactly as the kernel rounds
them (fp16 x fp16 products are exact in the fp32 accumulator), so the only difference left is the
summation order: tolerance 2e-5 of the output scale.  Layers on the 3-term split (all layers in f16x3, the transposed
convs in f16tc) are compared against the UNROUNDED fp32 conv at the same 2e-5: the split is FP32-equivalent.  This isolates descriptor / tap-shift /
pipeline bugs from the end-to-end fp16 error budget.
"""
import pytest
import torch
import torch.nn.functional as F

import gan_oracle as go
import ref_init as ri

pytestmark = pytest.mark.gpu


def _make(precision):
    from mockingbird_b200.vocoder.hifigan.models import Generator

    sd = ri.rescale_variance_preserving(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_16K, 0), 1.0)
    g = Generator(ri.HIFIGAN_CONFIG_16K, precision=precision).cuda()
    g.load_state_dict(sd)
    g.eval()
    g.remove_weight_norm()
    return g, sd


@pytest.fixture(scope="module")
def gen():
    return _make("f16tc")


@pytest.fixture(scope="module")
def gen_x3():
    return _make("f16x3")


def _is_x3(name, precision):
    """layers that run the FP32-equivalent 3-term split: all of them in f16x3; the serial transposed convs in f16tc"""
    return precision == "f16x3" or name.startswith("ups.") or name.startswith("cond_up.")


def _parse(info):
    d = dict(tok.split("=") for tok in info.split() if "=" in tok)
    return info.split()[1], {k: int(v) for k, v in d.items()}


def _layer_cases(g):
    """first conv of every distinct (cin, cout, k, dil, stride) signature"""
    seen, out = set(), []
    for i in range(g.num_layers()):
        name, d = _parse(g.layer_info(i))
        key = (d["cin"], d["cout"], d["k"], d["dil"], d["stride"], d["res"])
        if key in seen:
            continue
        seen.add(key)
        out.append(i)
    return out


def _reference(name, d, sd, x, res, q):
    w, b = sd[name + ".weight"], sd[name + ".bias"]
    slope = 1.0 if name == "conv_pre" else (0.01 if name == "conv_post" else 0.1)
    xa = F.leaky_relu(x, slope) if slope != 1.0 else x
    if q:
        xa, w = go.quant_fp16(xa), go.quant_fp16(w)
    if name.startswith("ups."):
        u = d["stride"]
        y = F.conv_transpose1d(xa, w, b, u, u // 2 + u % 2, u % 2)
    else:
        y = F.conv1d(xa, w, b, 1, go.get_padding(d["k"], d["dil"]), d["dil"])
    if res is not None:
        y = y + res
    if name == "conv_post":
        y = torch.tanh(y)
    return y


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("L", [300, 128, 1])
def test_every_layer_signature(gen, gen_x3, L, precision):
    g, sd = gen if precision == "f16tc" else gen_x3
    failures = []
    for i in _layer_cases(g):
        name, d = _parse(g.layer_info(i))
        B = 2
        gen_ = torch.Generator().manual_seed(1000 + i)
        x = torch.randn(B, d["cin"], L, generator=gen_)
        Lout = L * d["stride"]
        res = torch.randn(B, d["cout"], Lout, generator=gen_) if d["res"] else None
        y = g.debug_layer(i, x.cuda(), res.cuda() if res is not None else None, Lout).cpu()
        on_tc = name not in ("conv_pre", "conv_post")
        ref = _reference(name, d, sd, x, res, q=on_tc and not _is_x3(name, precision))
        err = float((y - ref).abs().max() / ref.abs().max())
        if not (err <= 2e-5):
            failures.append((i, name, d, err))
    assert not failures, failures


def test_tc_layer_is_actually_fp16(gen):
    """sanity: against the UNquantised fp32 conv the tensor-core layer shows fp16-sized error
    (so the test above really exercises the fp16 path and not an FP32 fallback)."""
    g, sd = gen
    idx = [i for i in range(g.num_layers()) if "resblocks.0.convs1.0" in g.layer_info(i)][0]
    name, d = _parse(g.layer_info(idx))
    x = torch.randn(1, d["cin"], 256, generator=torch.Generator().manual_seed(5))
    y = g.debug_layer(idx, x.cuda(), None, 256).cpu()
    ref32 = _reference(name, d, sd, x, None, q=False)
    err = float((y - ref32).abs().max() / ref32.abs().max())
    assert 1e-5 < err < 3e-3, err
