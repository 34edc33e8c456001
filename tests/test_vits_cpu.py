"""VITS host layer without a GPU: config validation, the ragged plan, the argument errors, the seeded weights against the
reference's parameter table, and the goldens' own consistency."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "synth_weights"))
import ref_init as ri  # noqa: E402

from mockingbird_b200 import _lib  # noqa: E402
from mockingbird_b200.synthesizer.models.vits import Vits  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"


def test_config_validation():
    with pytest.raises(ValueError, match="n_speakers == 1"):
        Vits(**dict(ri.VITS_TOY, n_speakers=1))
    with pytest.raises(ValueError, match="gin_channels"):
        Vits(**dict(ri.VITS_TOY, gin_channels=0))
    with pytest.raises(ValueError, match="precision"):
        Vits(**ri.VITS_TOY, precision="bf16")
    with pytest.raises(_lib.MbError, match="kernel_size"):
        Vits(**dict(ri.VITS_TOY, kernel_size=4))
    with pytest.raises(_lib.MbError, match="n_heads"):
        Vits(**dict(ri.VITS_TOY, n_heads=3))
    with pytest.raises(_lib.MbError, match="upsample"):
        Vits(**dict(ri.VITS_TOY, upsample_kernel_sizes=[7, 4]))
    v = Vits(**ri.VITS_CONFIG)
    assert v.hop == 256


def test_error_cases_before_any_device_work():
    v = Vits(**ri.VITS_TOY)
    x = torch.tensor([[1, 2, 3]])
    emo = torch.zeros(1, 1024)
    with pytest.raises(ValueError, match="emo"):
        v.infer(x, [3], sid=[0], emo=None)
    with pytest.raises(ValueError, match="speaker id"):
        v.infer(x, [3], sid=[3], emo=emo)
    with pytest.raises(ValueError, match="needs sid"):
        v.infer(x, [3], sid=None, emo=emo)
    with pytest.raises(ValueError, match="token id"):
        v.infer(torch.tensor([[1, 20]]), [2], sid=[0], emo=emo)
    with pytest.raises(ValueError, match="x_lengths"):
        v.infer(x, [4], sid=[0], emo=emo)
    with pytest.raises(ValueError, match="empty"):
        v.infer_many([[1, 2], []], [0, 0], torch.zeros(2, 1024), [1, 2])
    with pytest.raises(ValueError, match="seeds"):
        v.infer_many([[1, 2]], [0], torch.zeros(1, 1024), [1, 2])


def test_ragged_plan():
    plan = Vits.many_plan([3, 9, 5, 9, 1], 2)
    assert plan == [[1, 3], [2, 0], [4]]
    assert sorted(i for b in Vits.many_plan(list(range(37)), 16) for i in b) == list(range(37))


def test_weight_table_matches_reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_harness

    if not ref_harness.reference_available():
        pytest.skip("the reference tree is not here")
    import make_golden_vits as mg

    for cfg in (ri.VITS_TOY, ri.VITS_CONFIG, dict(ri.VITS_CONFIG, use_sdp=False), ri.VITS_TOY_1SPK):
        sd = ri.vits_state_dict(cfg, 0)
        m = mg.build_vits(cfg, sd)
        ref = {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.startswith("enc_q.") and not k.startswith("dp.post_")}
        assert ref == {k: tuple(v.shape) for k, v in sd.items()}


@pytest.mark.parametrize("name", ["toy", "full_sdp", "full_dp", "toy_1spk"])
def test_golden_consistency(name):
    g = np.load(GOLDEN / f"vits_{name}.npz")
    attn = g["attn"][:, 0]
    assert (attn.sum(1).astype(np.int32) == g["w_ceil"] * (np.arange(g["x"].shape[1])[None] < g["x_lengths"][:, None])).all()
    assert (attn.sum((1, 2)).astype(np.int32) == np.maximum(g["w_ceil"].sum(1), 0)).all()
    assert g["duration_margin"] >= 1e-3
    assert g["y_lengths"].max() == attn.shape[1]


CASE_CFG = {"toy": ri.VITS_TOY, "full_sdp": ri.VITS_CONFIG, "full_dp": dict(ri.VITS_CONFIG, use_sdp=False), "toy_1spk": ri.VITS_TOY_1SPK}


@pytest.mark.parametrize("name", ["toy", "full_sdp", "full_dp", "toy_1spk"])
def test_float64_restatement_against_goldens(name):
    """oracle/vits_oracle.infer on the goldens' inputs and noise against what the live reference recorded"""
    sys.path.insert(0, str(ROOT / "oracle"))
    import vits_oracle as vo

    g = np.load(GOLDEN / f"vits_{name}.npz")
    cfg = CASE_CFG[name]
    sd = ri.vits_state_dict(cfg, int(g["seed"]))
    with torch.no_grad():
        r = vo.infer(sd, cfg, torch.from_numpy(g["x"]), g["x_lengths"], g["sid"], g["emo"], g["sdp_noise"], torch.from_numpy(g["eps"]).double(),
                     float(g["noise_scale"]), float(g["noise_scale_w"]), float(g["length_scale"]), int(g["max_len"]) or None)
    mask = np.arange(g["x"].shape[1])[None] < g["x_lengths"][:, None]
    w = r["w"].numpy()[mask]
    assert np.abs(w - np.round(w)).min() >= 1e-3  # the float64 durations keep the margin the golden maker recorded
    assert np.array_equal(r["w_ceil"].numpy() * mask, g["w_ceil"] * mask)
    assert np.array_equal(r["y_lengths"].numpy(), g["y_lengths"])
    assert np.array_equal(r["attn"].numpy(), g["attn"])

    def rel(a, b):
        return float(np.abs(a.numpy() - b).max() / np.abs(b).max())

    for k in ("m_p", "logs_p", "m_p_y", "logs_p_y", "z_p", "z"):
        assert rel(r[k], g[k]) <= 1e-5, (k, rel(r[k], g[k]))
    assert r["o"].shape == g["o"].shape
    assert rel(r["o"], g["o"]) <= 1e-5, rel(r["o"], g["o"])


def _golden_case(name):
    sys.path.insert(0, str(ROOT / "oracle"))
    import vits_oracle as vo

    g = np.load(GOLDEN / f"vits_{name}.npz")
    cfg = CASE_CFG[name]
    return vo, g, cfg, ri.vits_state_dict(cfg, int(g["seed"]))


@pytest.mark.parametrize("name", ["toy", "full_sdp", "full_dp", "toy_1spk"])
def test_oracle_stages_compose_to_the_whole_chain(name):
    """the stage functions the kernel tests call (text_encoder_layer, logw, coupling_reverse), composed by hand on the goldens'
    inputs, give the whole-chain functions bit for bit, so the golden pin above covers them"""
    vo, g, cfg, sd = _golden_case(name)
    lens = torch.as_tensor(g["x_lengths"]).long()
    x = torch.from_numpy(g["x"])
    T = x.shape[1]
    m = vo.mask_of(lens, T)
    with torch.no_grad():
        h_ref, m_p, logs_p = vo.text_encoder(sd, cfg, x, lens, g["emo"])
        e = vo._d(g["emo"]) @ vo._d(sd["enc_p.emo_proj.weight"]).T + vo._d(sd["enc_p.emo_proj.bias"])
        h = (vo._d(sd["enc_p.emb.weight"])[x.long()] * np.sqrt(cfg["hidden_channels"]) + e[:, None, :]).transpose(1, 2) * m
        for l in range(cfg["n_layers"]):
            h = vo.text_encoder_layer(sd, cfg, l, h, lens, l == cfg["n_layers"] - 1)
        assert torch.equal(h, h_ref)
        gv = vo._d(sd["emb_g.weight"])[torch.as_tensor(g["sid"]).long()] if cfg["n_speakers"] > 1 else None
        lw = vo.logw(sd, cfg, h, lens, gv, g["sdp_noise"], float(g["noise_scale_w"]))
        ls = float(g["length_scale"])
        assert lw.shape == (x.shape[0], 1, T) and (lw * (1 - m) == 0).all()
        assert torch.equal(torch.exp(lw) * m * ls, vo.durations(sd, cfg, h, lens, gv, g["sdp_noise"], float(g["noise_scale_w"]), ls))
        z_p = torch.from_numpy(g["z_p"]).double()
        y_len = torch.as_tensor(g["y_lengths"]).long()
        z = z_p
        for f in (3, 2, 1, 0):
            z = vo.coupling_reverse(sd, f, torch.flip(z, [1]), y_len, gv)
        assert torch.equal(z, vo.flow_reverse(sd, z_p, y_len, gv))


def test_banded_attention_equals_the_dense_statement():
    """vo.rel_attention adds the relative terms on the 2W+1 diagonals; the dense statement builds the [T, T, dk] relative
    embeddings, zero outside the window"""
    sys.path.insert(0, str(ROOT / "oracle"))
    import vits_oracle as vo

    g = torch.Generator().manual_seed(0)
    for T, nh, H, lens in ((1, 2, 16, [1, 1]), (5, 2, 16, [5, 3]), (9, 3, 24, [9, 1]), (40, 1, 32, [40, 17])):
        q, k, v = (torch.randn(2, H, T, generator=g, dtype=torch.float64) for _ in range(3))
        erk, erv = torch.randn(1, 9, H // nh, generator=g), torch.randn(1, 9, H // nh, generator=g)
        dk = H // nh
        qh, kh, vh = (a.view(2, nh, dk, T).transpose(2, 3) for a in (q / np.sqrt(dk), k, v))
        rel = torch.arange(T)[None, :] - torch.arange(T)[:, None]
        inside = (rel.abs() <= vo.WINDOW)[..., None]
        idx = rel.clamp(-vo.WINDOW, vo.WINDOW) + vo.WINDOW
        rk, rv = erk.double()[0][idx] * inside, erv.double()[0][idx] * inside
        sc = qh @ kh.transpose(2, 3) + torch.einsum("bhtd,tsd->bhts", qh, rk)
        mk = vo.mask_of(lens, T)[:, 0]
        sc = torch.where((mk[:, None, :, None] * mk[:, None, None, :]) > 0, sc, torch.full_like(sc, -1e4))
        p = torch.softmax(sc, -1)
        dense = (p @ vh + torch.einsum("bhts,tsd->bhtd", p, rv)).transpose(2, 3).reshape(2, H, T)
        got = vo.rel_attention(q, k, v, erk, erv, torch.tensor(lens), nh)
        assert (got - dense).abs().max() <= 1e-13 * dense.abs().max(), T
