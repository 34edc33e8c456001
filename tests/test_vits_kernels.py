"""The VITS kernel stages launch by launch (mb_vits_debug, mb_vits_decode) against the float64 restatement in
oracle/vits_oracle.py, on seeded weights: the spline inverse across its bins, at bin edges and in both tails; relative
attention below, at and above the window with padded keys; a WN layer with and without g; DDSConv; the path expansion with
zero-duration tokens; the decoder on its own."""
import ctypes as C
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "synth_weights"))
sys.path.insert(0, str(ROOT / "oracle"))
import ref_init as ri  # noqa: E402
import vits_oracle as vo  # noqa: E402

from mockingbird_b200 import _lib  # noqa: E402
from mockingbird_b200.synthesizer.models.vits import Vits  # noqa: E402

pytestmark = pytest.mark.gpu
_models = {}


def model(cfg_name, precision="fp32"):
    key = (cfg_name, precision)
    if key not in _models:
        cfg = {"toy": ri.VITS_TOY, "full": ri.VITS_CONFIG, "toy_1spk": ri.VITS_TOY_1SPK}[cfg_name]
        sd = ri.vits_state_dict(cfg, 21)
        m = Vits(**cfg, precision=precision)
        m.load_state_dict(sd)
        m.cuda()
        m.remove_weight_norm()
        _models[key] = (m, cfg, sd)
    return _models[key]


def debug(m, kind, B, T, x, x2=None, x3=None, y=None, y2=None, lengths=None, index=0, sub=0, c0=0, c1=0):
    s = _lib.VitsDebugSpec()
    s.kind, s.batch, s.frames, s.index, s.sub, s.c0, s.c1 = _lib.MB_VITS_DBG[kind], B, T, index, sub, c0, c1
    for f, t in (("lengths", lengths), ("x", x), ("x2", x2), ("x3", x3), ("y", y), ("y2", y2)):
        setattr(s, f, t.data_ptr() if t is not None else None)
    L = _lib.lib()
    ws = torch.empty(int(L.mb_vits_debug_workspace_bytes(m._handle, C.byref(s))), dtype=torch.uint8, device="cuda")
    _lib.check(L.mb_vits_debug(m._handle, C.byref(s), C.c_void_p(ws.data_ptr()), ws.numel(),
                               C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_spline_across_bins_edges_and_tails():
    m, cfg, sd = model("toy")
    H, B, T = cfg["hidden_channels"], 2, 96
    g = torch.Generator().manual_seed(1)
    h = torch.randn(B, H, T, generator=g) * 2
    lens = torch.tensor([T, T - 7], dtype=torch.int32)
    for f in (3, 5, 7):
        # the knots of every frame, in float64, to place inputs exactly on bin edges
        p = (vo.conv(sd, f"dp.flows.{f}.proj", h.double()) * vo.mask_of(lens, T)).transpose(1, 2)
        p = torch.cat([p[..., :20] / math.sqrt(H), p[..., 20:]], -1)
        w = 1e-3 + (1 - 1e-2) * torch.softmax(p[..., 10:20], -1)
        knots = torch.cat([torch.zeros(B, T, 1, dtype=torch.float64), torch.cumsum(w, -1)], -1) * 10 - 5
        x1 = torch.linspace(-7.5, 7.5, T).repeat(B, 1).double()
        x1[:, ::3] = knots[:, ::3, 1:10].gather(-1, (torch.arange(0, T, 3) % 9)[None, :, None].expand(B, -1, 1))[..., 0]
        z = torch.stack([torch.randn(B, T, generator=g).double(), x1], 1).float()
        z[:, 1, 1] = 5.0
        z[:, 1, 2] = -5.0
        for c0, c1 in ((0, 1), (1, 0)):
            zz = z if c1 == 1 else z.flip(1)
            y = torch.empty(B, 2, T, device="cuda")
            debug(m, "spline", B, T, h.cuda(), zz.cuda(), y=y, lengths=lens.cuda(), index=f, c0=c0, c1=c1)
            ref = vo.convflow_spline(sd, f, h.double(), zz.double(), lens, c0, c1)
            assert (y.cpu().double() - ref).abs().max() <= 2e-5, (f, c0)
        inside = z[:, 1].abs() <= 5
        assert (~inside).any(dim=1).all() and (z[:, 1] > 5).any() and (z[:, 1] < -5).any()  # both tails
        bins = ((z[:, 1, :, None].double() >= knots[..., :10]).sum(-1) - 1)[inside]
        assert set(bins.tolist()) >= set(range(10))


@pytest.mark.parametrize("T,lens", [(3, [3, 2]), (4, [4, 1]), (5, [5, 3]), (9, [9, 6]), (40, [40, 17])])
def test_relative_attention(T, lens):
    m, cfg, sd = model("full")
    H = cfg["hidden_channels"]
    g = torch.Generator().manual_seed(T)
    q, k, v = (torch.randn(2, H, T, generator=g) for _ in range(3))
    lens_t = torch.tensor(lens, dtype=torch.int32)
    for layer in (0, 5):
        y = torch.empty(2, H, T, device="cuda")
        debug(m, "attn", 2, T, q.cuda(), k.cuda(), v.cuda(), y=y, lengths=lens_t.cuda(), index=layer)
        a = f"enc_p.encoder.attn_layers.{layer}"
        ref = vo.rel_attention(q.double(), k.double(), v.double(), sd[a + ".emb_rel_k"], sd[a + ".emb_rel_v"], lens_t, cfg["n_heads"])
        assert rel(y, ref) <= 1e-5, (T, layer, rel(y, ref))


@pytest.mark.parametrize("with_g", [True, False])
@pytest.mark.parametrize("sub", [0, 2, 3])
def test_wn_layer(with_g, sub):
    m, cfg, sd = model("toy")
    H, G, B, T = cfg["hidden_channels"], cfg["gin_channels"], 2, 77
    g = torch.Generator().manual_seed(sub)
    lens = torch.tensor([T, 50], dtype=torch.int32)
    h = torch.randn(B, H, T, generator=g) * vo.mask_of(lens, T).float()
    skip = torch.randn(B, H, T, generator=g)
    gv = torch.randn(B, G, generator=g) if with_g else None
    y, y2 = torch.empty(B, H, T, device="cuda"), skip.clone().cuda()
    debug(m, "wn", B, T, h.cuda(), gv.cuda() if with_g else None, y=y, y2=y2, lengths=lens.cuda(), index=1, sub=sub)
    e = "flow.flows.2.enc."
    cond = vo.conv(sd, e + "cond_layer", gv.double()[:, :, None])[:, :, 0] if with_g else None
    rh, rs = vo.wn_layer(sd, e, sub, h.double(), None if sub == 0 else skip.double(), cond, lens)
    assert rel(y, rh) <= 1e-5 and rel(y2, rs) <= 1e-5


@pytest.mark.parametrize("index", [0, 5])
def test_ddsconv(index):
    m, cfg, sd = model("toy")
    H, B, T = cfg["hidden_channels"], 3, 61
    lens = torch.tensor([61, 30, 4], dtype=torch.int32)
    x = torch.randn(B, H, T, generator=torch.Generator().manual_seed(index))
    y = torch.empty(B, H, T, device="cuda")
    debug(m, "ddsconv", B, T, x.cuda(), y=y, lengths=lens.cuda(), index=index)
    ref = vo.ddsconv(sd, "dp.convs." if index == 0 else f"dp.flows.{index}.convs.", x.double(), lens)
    assert rel(y, ref) <= 1e-5


def test_path_expansion_with_zero_duration_tokens():
    m, cfg, sd = model("toy")
    I, B, Tx = cfg["inter_channels"], 3, 8
    g = torch.Generator().manual_seed(4)
    w_ceil = torch.tensor([[2, 0, 3, 0, 0, 1, 4, 0], [0, 0, 5, 1, 9, 9, 9, 9], [0, 0, 0, 0, 0, 0, 0, 0]], dtype=torch.int32)
    x_len = torch.tensor([8, 4, 6], dtype=torch.int32)
    m_p, logs_p = torch.randn(B, I, Tx, generator=g), torch.randn(B, I, Tx, generator=g) * 0.3
    attn_r, z_p_r, m_y_r, l_y_r, y_len = vo.expand(m_p.double(), logs_p.double(), w_ceil, x_len,
                                                   torch.zeros(B, I, 12, dtype=torch.float64), 0.0)
    assert y_len.tolist() == [10, 6, 1]  # an utterance of zero-duration tokens still decodes one frame
    eps = torch.randn(B, I, 12, generator=g)
    _, z_p_r, _, _, _ = vo.expand(m_p.double(), logs_p.double(), w_ceil, x_len, eps.double(), 0.667)
    sid = torch.tensor([0, 1, 2], dtype=torch.int32, device="cuda")
    with torch.cuda.device(m._device):
        _, attn, z_p, _, m_y, l_y = m._decode(m_p.cuda(), logs_p.cuda(), w_ceil.cuda(), x_len.cuda(), sid, eps.cuda(), 0.667, 12, True, True)
    assert torch.equal(attn.cpu().double(), attn_r)
    assert torch.equal(m_y.cpu().double(), m_y_r.float().double()) and torch.equal(l_y.cpu().double(), l_y_r.float().double())
    assert rel(z_p, z_p_r) <= 1e-6


@pytest.mark.parametrize("cfg_name", ["toy", "toy_1spk", "full"])
@pytest.mark.parametrize("precision,tol", [("fp32", 3e-6), ("f16x3", 2e-5), ("f16tc", 1e-3)])
def test_decoder_alone(cfg_name, precision, tol):
    """the MB_GAN_VITS decoder with cond(g) folded into conv_pre, on its own input, at the decoder bounds of DESIGN.md 4l"""
    m, cfg, sd = model(cfg_name, precision)
    I, B, T = cfg["inter_channels"], 2, 24
    z = torch.randn(B, I, T, generator=torch.Generator().manual_seed(9))
    sid = torch.tensor([1, 0], dtype=torch.int32)
    y = torch.empty(B, 1, T * m.hop, device="cuda")
    multi = cfg["n_speakers"] > 1
    debug(m, "decoder", B, T, z.cuda(), sid.cuda() if multi else None, y=y)
    g = torch.as_tensor(sd["emb_g.weight"]).double()[sid.long()] if multi else None
    ref = vo.decoder(sd, cfg, z.double(), g)
    e = rel(y, ref)
    print(cfg_name, precision, "decoder max_rel", e)
    assert e <= tol, e
