"""The PPG extractor on the GPU (mockingbird_b200.ppg_extractor, mb_ppgx_*): parity with the golden vectors recorded
from the live reference, every block's output against the plain-torch restatement, every small-config variant, padded
batches bitwise equal to B = 1 calls, the positional-table high-water mark, load_model and the voice-conversion chain."""
import numpy as np
import pytest
import torch

import gan_oracle as go
import golden_io
import ppgx_oracle as po
import ref_init as ri
from mockingbird_b200.ppg_extractor import PPGModel, build_model

pytestmark = pytest.mark.gpu

TOL = 1e-3


@pytest.fixture(scope="module")
def golden(golden_dir):
    return golden_io.load(golden_dir / "ppgx_seed0.npz")


def model(cfg, seed=0):
    m = build_model(cfg)
    m.load_state_dict(ri.ppg_extractor_state_dict(cfg, seed))
    return m.cuda().eval()


@pytest.fixture(scope="module")
def std():
    return model(ri.PPGX_CONFIG)


def run1(m, wav):
    w = torch.from_numpy(wav)
    return m(w[None], torch.LongTensor([w.numel()]))[0].cpu()


def test_golden_stand_in(golden, std):
    for case in ("a", "b"):
        out = run1(std, golden[case + "_wav"])
        e = go.rel_errors(out, torch.from_numpy(golden[case + "_out"]))
        print(f"ppgx golden {case}: {e}")
        assert out.shape == golden[case + "_out"].shape
        assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, (case, e)


def test_taps(golden, std):
    w = torch.from_numpy(golden["a_wav"])
    out, taps = std.forward(w[None], torch.LongTensor([w.numel()]), return_taps=True)
    assert taps.shape == (17, 1, 301, 144)
    for i, ref in zip(golden["a_tap_index"], golden["a_taps"]):
        e = go.rel_errors(taps[i, 0].cpu(), torch.from_numpy(ref))
        print(f"ppgx golden tap {i}: {e}")
        assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, (i, e)
    _, ref_taps = po.forward(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0), ri.PPGX_CONFIG, w, taps=True)
    for i, ref in enumerate(ref_taps):
        e = go.rel_errors(taps[i, 0].cpu(), ref)
        assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, (i, e)


@pytest.mark.parametrize("name", ["small"] + list(ri.PPGX_SMALL_VARIANTS))
def test_small_variants(golden, name):
    cfg = ri.PPGX_CONFIG_SMALL if name == "small" else ri.PPGX_SMALL_VARIANTS[name]
    out = run1(model(cfg), golden["v_wav"])
    ref = torch.from_numpy(golden[f"v_{name}_out"])
    e = go.rel_errors(out, ref)
    print(f"ppgx variant {name}: {e}")
    assert out.shape == ref.shape and e["max_rel"] <= TOL and e["rms_rel"] <= TOL, e


def _wavs(n, seed, lo=3000, hi=20000):
    g = np.random.RandomState(seed)
    return [(0.3 * g.randn(int(g.randint(lo, hi)))).astype(np.float32) for _ in range(n)]


@pytest.mark.parametrize("cfg_name,rows", [("std", 1), ("std", 5), ("small", 128), ("small", 130)])
def test_batch_rows_bitwise_equal_b1(std, cfg_name, rows):
    m = std if cfg_name == "std" else model(ri.PPGX_CONFIG_SMALL)
    wavs = _wavs(rows, rows, hi=20000 if rows < 100 else 6000)
    outs = m.extract_batch(wavs)
    for w, o in zip(wavs, outs):
        assert o.shape == (m.num_frames(len(w)), m.d_model)
        assert torch.isfinite(o).all()
    for i in sorted({0, rows // 2, rows - 1}):
        one = run1(m, wavs[i])
        assert torch.equal(outs[i].cpu(), one), i
    if rows <= 5:
        n_max = max(len(w) for w in wavs)
        pad = torch.zeros(rows, n_max)
        for r, w in enumerate(wavs):
            pad[r, :len(w)] = torch.from_numpy(w)
        out = m(pad, torch.LongTensor([len(w) for w in wavs])).cpu()
        for r, w in enumerate(wavs):
            t = m.num_frames(len(w))
            assert torch.equal(out[r, :t], outs[r].cpu()) and not out[r, t:].any()


def test_pe_len_high_water_mark(golden):
    m = model(ri.PPGX_CONFIG_SMALL)
    wav = po_synthetic(int(golden["long_n"]), int(golden["long_wav_seed"]))
    out = run1(m, wav)
    assert m.pe_len == int(golden["long_pe_len"]) == out.shape[0] > 5000
    for k, rows in (("long_head", out[:64]), ("long_tail", out[-64:])):
        e = go.rel_errors(rows, torch.from_numpy(golden[k]))
        assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, (k, e)
    short = run1(m, golden["short_wav"])
    assert m.pe_len == int(golden["short_pe_len"])
    e = go.rel_errors(short, torch.from_numpy(golden["short_out"]))
    assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, e
    # a fresh instance keeps pe_len 5000: a different relative-position table, outside the tolerance of the golden
    fresh = run1(model(ri.PPGX_CONFIG_SMALL), golden["short_wav"])
    e = go.rel_errors(fresh, torch.from_numpy(golden["short_out"]))
    assert e["max_rel"] > TOL, e


def po_synthetic(n, seed):
    """make_golden_ppgx.synthetic_wav (the long case's wav is regenerated, not stored)"""
    g = np.random.RandomState(seed)
    t = np.arange(n) / 16000.0
    x = 0.3 * np.sin(2 * np.pi * 220 * t) + 0.2 * np.sin(2 * np.pi * 1250 * t + 0.3) + 0.1 * np.sin(2 * np.pi * 3100 * t)
    x += 0.1 * np.sin(2 * np.pi * (300 + 800 * t) * t) + 0.05 * g.randn(n)
    x[int(0.40 * n):int(0.45 * n)] = 0.0
    return x.astype(np.float32)


def test_load_model(tmp_path, golden):
    import yaml

    from mockingbird_b200 import ppg_extractor as E

    sd = ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0)
    torch.save({k: v for k, v in sd.items() if k.startswith("encoder.")}, tmp_path / "ppg.pt")
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(ri.PPGX_CONFIG))
    m = E.load_model(tmp_path / "ppg.pt")
    assert E._model is m and isinstance(m, PPGModel) and E._device.type == "cuda"
    out = m.extract_from_wav(golden["a_wav"])[0].cpu()
    e = go.rel_errors(out, torch.from_numpy(golden["a_out"]))
    assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, e


def test_vc_chain_on_device(golden, std):
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2
    from mockingbird_b200.vocoder.hifigan.models import Generator

    ppg = std.extract_from_wav(golden["a_wav"])
    assert ppg.is_cuda and ppg.shape == (1, 301, 144)
    T = ppg.shape[1]
    lf0 = torch.stack([torch.linspace(4.5, 5.5, T), (torch.arange(T) % 7 > 1).float()], -1)[None].cuda()
    dec = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    dec.load_state_dict(ri.ppg2mel_state_dict(0))
    dec.eval()
    mel, post, align = dec.inference(ppg, lf0, torch.randn(1, 256).cuda(), seed=3)
    assert post.is_cuda and post.shape[1] == 80 and post.shape[0] == 2 * align.shape[0] and align.shape[1] == T // 4
    voc = Generator(ri.HIFIGAN_CONFIG_24K).cuda()
    voc.load_state_dict(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0))
    voc.eval()
    voc.remove_weight_norm()
    wav = voc(post.T[None].contiguous())
    assert wav.is_cuda and wav.shape == (1, 1, 240 * post.shape[0]) and torch.isfinite(wav).all()
