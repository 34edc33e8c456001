"""Harvest on the H100 (mb_f0_*) against the float64 restatement (oracle/harvest_oracle.py), stage by stage through the
debug outputs and on the final contour; ragged batches bitwise against single calls; the voice-conversion lf0 features on
device F0."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "oracle"))

import harvest_oracle as ho  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(ROOT / "tests" / "golden" / "f0_seed0.npz")
CLIPS = [GOLDEN[f"clip_{i}"] for i in range(len([k for k in GOLDEN.files if k.startswith("clip_")]))]
RTOL = 1e-9


def _fu():
    from mockingbird_b200 import f0_utils

    return f0_utils


def _close(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) <= RTOL * np.maximum(np.abs(a), np.abs(b))


def _margins(st):
    """smallest relative distance of a thresholded decision of the restatement to its threshold"""
    sc = st["scores"][st["refined"] > 0]
    m = [np.min(np.abs(sc / 2.5 - 1.0))] if sc.size else []
    rf = st["refined"]
    if rf.shape[0] >= 3 and rf.shape[1]:
        ref = rf[1:-1]
        with np.errstate(divide="ignore", invalid="ignore"):
            for nb in (rf[2:], rf[:-2]):
                e = np.abs(ref[:, :, None] - nb[:, None, :]) / ref[:, :, None]
                e = e[ref > 0]
                if e.size:
                    m.append(np.min(np.abs(e / 0.05 - 1.0)))
    return min(m) if m else float("inf")


def _stage_check(x, dbg, i):
    st = ho.harvest_stages(x)
    assert np.array_equal(dbg["raw_count"][i], st["raw_count"])
    assert np.array_equal(dbg["official_count"][i], st["official_count"])
    S = st["refined"].shape[1]
    rf, rs = dbg["refined"][i], dbg["scores"][i]
    assert np.all(rf[:, S:] == 0) and np.all(rs[:, S:] == 0)
    assert np.array_equal(rf[:, :S] > 0, st["refined"] > 0)
    assert np.all(_close(rf[:, :S], st["refined"])) and np.all(_close(rs[:, :S], st["scores"]))
    assert np.array_equal(dbg["contour"][i] > 0, st["contour"] > 0)
    assert np.all(_close(dbg["contour"][i], st["contour"]))
    return st


def test_stages_and_contour_against_restatement():
    fu = _fu()
    x10 = ho.speechlike(1234, 160000)
    clips = CLIPS + [x10]
    dbg = {}
    out = fu.harvest_many(clips, debug=dbg)
    worst = float("inf")
    for i, x in enumerate(clips):
        st = _stage_check(x, dbg, i)
        assert np.array_equal(out[i] > 0, st["f0"] > 0), f"clip {i}: voicing differs"
        assert np.all(_close(out[i], st["f0"])), f"clip {i}: max rel {np.max(np.abs(out[i] - st['f0']) / np.maximum(st['f0'], 1e-300))}"
        worst = min(worst, _margins(st))
    print(f"smallest relative margin of a thresholded decision (score 2.5, 5 % neighbour rule): {worst:.3e}")


def test_compute_f0_on_golden_clips():
    fu = _fu()
    for i, x in enumerate(CLIPS):
        f0 = fu.compute_f0(x)
        ref = GOLDEN[f"f0_{i}"]
        assert f0.dtype == np.float32 and f0.shape == ref.shape
        assert np.array_equal(f0 > 0, ref > 0)
        assert np.all(np.abs(f0.astype(np.float64) - ref) <= 1e-6 * ref + 1e-30)
        assert np.array_equal(fu.compute_f0(x.astype(np.float64)), f0)


@pytest.mark.parametrize("b", [1, 7, 64])
def test_batches_are_bitwise_single_calls(b):
    fu = _fu()
    rng = np.random.default_rng(b)
    lengths = sorted(int(v) for v in rng.integers(1, 48000, size=b))
    lengths[0] = 1 if b > 1 else lengths[0]
    clips = [ho.speechlike(1000 + i, n) for i, n in enumerate(lengths)]
    single = [fu.compute_f0(c) for c in clips]
    for order in (np.arange(b), rng.permutation(b)):
        got = fu.compute_f0_many([clips[i] for i in order])
        for j, i in enumerate(order):
            assert got[j].dtype == np.float32 and np.array_equal(got[j], single[i]), f"clip {i} at row {j}"


def test_lf0uv_on_device_f0():
    fu = _fu()
    m, s = GOLDEN["mean_0"], GOLDEN["std_0"]
    many = fu.get_converted_lf0uv_many(CLIPS, [m] * len(CLIPS), [s] * len(CLIPS))
    for i, x in enumerate(CLIPS):
        one = fu.get_converted_lf0uv(x, m, s)
        assert np.array_equal(one, many[i])
        host = fu._lf0uv(fu.compute_f0(x), m, s, True)
        assert np.array_equal(one, host)
        ref = fu._lf0uv(ho.harvest(x)[0].astype(np.float32), m, s, True)
        assert np.array_equal(one[:, 1], ref[:, 1])
        assert np.allclose(one[:, 0], ref[:, 0], rtol=1e-6, atol=0)
        raw = fu.get_converted_lf0uv(x, m, s, convert=False)
        assert raw.shape == (len(fu.compute_f0(x)), 2)


def test_voice_conversion_chain_with_real_f0():
    """wav -> PPG -> lf0_uv from device F0 -> ppg2mel -> 24 kHz HiFi-GAN, with stand-in seeded weights"""
    import torch

    sys.path.insert(0, str(ROOT / "synth_weights"))
    import ref_init as ri
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2
    from mockingbird_b200.ppg_extractor import build_model
    from mockingbird_b200.vocoder.hifigan.models import Generator

    fu = _fu()
    m = build_model(ri.PPGX_CONFIG)
    m.load_state_dict(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0))
    m.cuda().eval()
    dec = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    dec.load_state_dict(ri.ppg2mel_state_dict(0))
    dec.eval()
    voc = Generator(ri.HIFIGAN_CONFIG_24K).cuda()
    voc.load_state_dict(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0))
    voc.eval()
    voc.remove_weight_norm()
    src = CLIPS[:3]
    with torch.no_grad():
        feats = m.extract_batch(src)
        lf0s = fu.get_converted_lf0uv_many(src, [GOLDEN["mean_0"]] * 3, [GOLDEN["std_0"]] * 3)
        utts = []
        for p, l in zip(feats, lf0s):
            n = min(p.shape[0], len(l))
            assert n == min(p.shape[0], fu.num_frames(len(src[len(utts)])))
            utts.append((p[:n], torch.from_numpy(l[:n]).float().cuda()))
        spk = torch.randn(3, 256, generator=torch.Generator().manual_seed(4))
        outs = dec.inference_batch(utts, spk, seed=3)
        for o in outs:
            mel = o[1].t()[None]
            wav = voc(mel)
            assert wav.shape[-1] == mel.shape[-1] * voc.hop
            assert torch.isfinite(wav).all()
