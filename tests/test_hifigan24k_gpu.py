"""GPU tests of the 24 kHz HiFi-GAN (nearest upsample + Conv1d per stage, hifigan/models.py:107-118), lowered to folded
polyphase tap convs: the library against the fixture recorded from the live reference, against the CPU oracle, through the
drop-in module protocol, and each folded upsampling layer alone against a float64 interpolate-and-conv reference.

Tolerances are those of tests/test_gan_gpu.py (max_rel and rms_rel): fp32 2e-5, f16x3 1e-4, f16tc 1e-3, auto 1e-3.
"""
import json

import numpy as np
import pytest
import torch

import gan_oracle as go
import hifigan24k_oracle as o24
import ref_init as ri
import tc_pair_oracle as po

pytestmark = pytest.mark.gpu

TOL = {"fp32": 2e-5, "f16tc": 1e-3, "f16x3": 1e-4, "auto": 1e-3}
PRECISIONS = ["fp32", "f16tc", "f16x3"]
CONFIGS = {"24k": ri.HIFIGAN_CONFIG_24K, "24k_u8": ri.HIFIGAN_CONFIG_24K_U8}
SLOPE = 0.1


@pytest.fixture(scope="module")
def sds():
    return {name: ri.hifigan_state_dict(cfg, 0) for name, cfg in CONFIGS.items()}


def _gen(name, precision, sd):
    from mockingbird_b200.vocoder.hifigan.models import Generator

    g = Generator(CONFIGS[name], precision=precision).cuda()
    g.load_state_dict(sd)
    g.eval()
    g.remove_weight_norm()
    return g


def _ok(e, precision):
    return e["max_rel"] <= TOL[precision] and e["rms_rel"] <= TOL[precision]


@pytest.mark.parametrize("precision", PRECISIONS)
def test_golden_small(golden_dir, sds, precision):
    z = np.load(golden_dir / "hifigan24k_seed0.npz")
    g = _gen("24k", precision, sds["24k"])
    wav = g(torch.from_numpy(z["mel_small"]).cuda()).cpu()
    assert wav.shape == (2, 1, 24 * 240)
    e = go.rel_errors(wav, torch.from_numpy(z["wav_small"]))
    print(precision, e)
    assert _ok(e, precision), e


@pytest.mark.parametrize("precision", PRECISIONS)
def test_golden_full_size_rows(golden_dir, sds, precision):
    """batch 32 x 256 frames (61 440 samples per row): rows 0 and 31 against the fixture, row 5 alone equals its batched row"""
    z = np.load(golden_dir / "hifigan24k_seed0.npz")
    g = _gen("24k", precision, sds["24k"])
    mel = torch.rand(32, 80, 256, generator=torch.Generator().manual_seed(2)) * 8 - 4
    wav = g(mel.cuda())
    assert wav.shape == (32, 1, 61440)
    pick = [int(i) for i in z["full_pick"]]
    e = go.rel_errors(wav[pick].cpu(), torch.from_numpy(z["wav_full"]))
    print(precision, e)
    assert _ok(e, precision), e
    alone = g(mel[5:6].cuda())
    assert torch.equal(alone[0], wav[5])


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", sorted(CONFIGS))
@pytest.mark.parametrize("B,T", [(1, 1), (1, 7), (3, 33), (2, 130)])
def test_vs_oracle_shapes(sds, name, precision, B, T):
    g = _gen(name, precision, sds[name])
    mel = torch.rand(B, 80, T, generator=torch.Generator().manual_seed(100 + T)) * 8 - 4
    with torch.no_grad():
        ref = o24.hifigan24k_forward(sds[name], CONFIGS[name], mel)
    wav = g(mel.cuda()).cpu()
    assert wav.shape == (B, 1, T * 240)
    e = go.rel_errors(wav, ref)
    assert _ok(e, precision), e


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_ragged_batch_equals_per_utterance(sds, name, precision):
    """padding is masked at every layer: each row equals its own batch-1 call, and is zero past its end"""
    g = _gen(name, precision, sds[name])
    lens = [40, 17, 33, 1]
    mel = torch.full((4, 80, 40), -4.0)
    for i, t in enumerate(lens):
        mel[i, :, :t] = torch.rand(80, t, generator=torch.Generator().manual_seed(i)) * 8 - 4
    wav = g(mel.cuda(), lengths=torch.tensor(lens, dtype=torch.int32)).cpu()
    for i, t in enumerate(lens):
        alone = g(mel[i:i + 1, :, :t].cuda()).cpu()
        assert torch.equal(wav[i:i + 1, :, : t * 240], alone), i
        if t < 40:
            assert float(wav[i, :, t * 240:].abs().max()) == 0.0, i
        with torch.no_grad():
            ref = o24.hifigan24k_forward(sds[name], CONFIGS[name], mel[i:i + 1, :, :t])
        e = go.rel_errors(alone, ref)
        assert _ok(e, precision), (i, e)


def test_auto_selection(sds):
    """the drop-in default decides f16tc vs f16x3 once at load time and reports its probe; either way it meets 1e-3"""
    g = _gen("24k", "auto", sds["24k"])
    c = g.calibration
    print("auto:", c)
    assert g.precision == c["selected"] in ("f16tc", "f16x3"), c
    assert (c["selected"] == "f16tc") == (c["max_rel"] <= g.AUTO_TOLERANCE and c["rms_rel"] <= g.AUTO_TOLERANCE), c
    mel = torch.rand(2, 80, 50, generator=torch.Generator().manual_seed(6)) * 8 - 4
    with torch.no_grad():
        ref = o24.hifigan24k_forward(sds["24k"], CONFIGS["24k"], mel)
    e = go.rel_errors(g(mel.cuda()).cpu(), ref)
    assert _ok(e, "auto"), e


def test_inference_module_protocol(tmp_path, sds):
    """hifigan/inference.py's protocol from files: a checkpoint with weight_g / weight_v keys and the 24 kHz json beside it"""
    from mockingbird_b200.vocoder.hifigan import inference as gan_vocoder

    sd0 = sds["24k"]
    raw = {}
    for k, v in sd0.items():
        if k.endswith(".weight"):
            base = k[: -len(".weight")]
            raw[base + ".weight_v"] = v * 3.0
            raw[base + ".weight_g"] = v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, 1, 1)  # dim 0: Cout of a Conv1d
        else:
            raw[k] = v
    assert "ups.0.1.weight_g" in raw
    torch.save({"generator": raw}, tmp_path / "g_02830000.pt")
    (tmp_path / "config.json").write_text(json.dumps(ri.HIFIGAN_CONFIG_24K))
    before = gan_vocoder._precision
    gan_vocoder.set_precision("fp32")
    try:
        gan_vocoder.load_model(tmp_path / "g_02830000.pt", verbose=False)
    finally:
        gan_vocoder.set_precision(before)
    assert gan_vocoder.is_loaded() and gan_vocoder.output_sample_rate == 24000
    mel = (torch.rand(80, 30, generator=torch.Generator().manual_seed(8)) * 8 - 4).numpy()
    wav, sr = gan_vocoder.infer_waveform(mel)
    assert sr == 24000 and wav.shape == (30 * 240,) and wav.dtype == np.float32
    with torch.no_grad():
        ref = o24.hifigan24k_forward(sd0, ri.HIFIGAN_CONFIG_24K, torch.from_numpy(mel)[None])
    assert go.rel_errors(torch.from_numpy(wav)[None, None], ref)["max_rel"] <= TOL["fp32"]
    many = gan_vocoder.infer_waveforms([mel[:, :11], mel, mel[:, :25]], batch_size=2)
    assert [w.shape[0] for w in many] == [11 * 240, 30 * 240, 25 * 240]
    assert np.array_equal(many[1], wav)
    gan_vocoder.generator = None


def _padded(sd, name, cin, cout):
    """checkpoint Conv1d weight / bias zero-padded to the plan's channel counts (the 16-channel stage runs with 32)"""
    w, b = sd[name + ".weight"], sd[name + ".bias"]
    wp = torch.zeros(cout, cin, w.shape[2])
    wp[: w.shape[0], : w.shape[1]] = w
    bp = torch.zeros(cout)
    bp[: b.shape[0]] = b
    return wp.cuda(), bp.cuda()


def _ups_layers(g):
    out = []
    for i in range(g.num_layers()):
        s = g.layer_info(i).split()
        if s[1].startswith("ups."):
            out.append((i, s[1], {k: int(v) for k, v in (t.split("=") for t in s[2:])}))
    return out


@pytest.mark.parametrize("ups_x3", [1, 0])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_each_folded_layer_alone(sds, name, ups_x3, monkeypatch):
    """every ups.{i}.1 as one tensor-core launch (mb_gan_debug_launch, with lengths) against float64 references rounded where the
    kernel rounds: the 3-term split (default) against interpolate + conv of the fp32 activation; the plain fp16 variant
    (MB_TC_UPS_X3=0) against the fold summed in fp32, rounded to fp16, applied to the fp16 activation"""
    monkeypatch.setenv("MB_TC_UPS_X3", str(ups_x3))
    g = _gen(name, "f16tc", sds[name])
    gen = torch.Generator().manual_seed(21)
    for i, lname, d in _ups_layers(g):
        p = g.tc_plan_info(i)
        assert p["use_tc"] == 1 and p["x3"] == ups_x3, (lname, p)
        u = d["stride"]
        Lin, vin = 300, [300, 123]
        B, Lout = 2, 300 * u
        valid = [n * u for n in vin]
        x = torch.randn(B, d["cin"], Lin, generator=gen).cuda() * po.row_mask(B, Lin, vin, "cuda").float()
        y, _, _, ln = g.debug_launch(i, x, lengths=torch.tensor(vin, dtype=torch.int32).cuda())
        assert ln[0]["kernel"] == (d["cout"], p["mt"], p["kc"], 0), (lname, ln, p)
        w, b = _padded(sds[name], lname, d["cin"], d["cout"])
        if ups_x3:
            a = po.act32(x, SLOPE)
            ref = torch.nn.functional.conv1d(o24.interpolate_nearest(a, u), w.double(), b.double(), padding=(d["k"] - 1) // 2)
        else:
            a = po.q16(po.act32(x, SLOPE))
            ref = o24.folded_forward(a, w, b, u, wround=po.q16)
        ref = ref * po.row_mask(B, Lout, valid, "cuda")
        bound = po.TOL * ref.abs().max() * po.row_mask(B, Lout, valid, "cuda")
        r = po.worst_ratio(y, ref, bound)
        print(name, lname, "x3" if ups_x3 else "f16", "worst |y - ref| / bound", round(r, 4))
        assert r <= 1.0, (lname, r)
