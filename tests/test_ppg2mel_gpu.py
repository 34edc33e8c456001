"""GPU tests of the voice-conversion mel decoder (mockingbird_b200.ppg2mel, mb_ppg2mel_*): the golden cases from the
live reference, padded batches against each row's own B = 1 call and the oracle, padding isolation, device-drawn
dropout, load_model, the ppg2mel -> HiFi-GAN chain and input validation."""
import numpy as np
import pytest
import torch

import golden_io
import ppg2mel_oracle as po
from ppg2mel_kernel_oracle import philox_keep as _philox_keep
import ref_init as ri

pytestmark = pytest.mark.gpu
CASES = ("a", "b", "c")
TOL = 1e-3


@pytest.fixture(scope="module")
def golden(golden_dir):
    return golden_io.load(golden_dir / "ppg2mel_seed0.npz")


def case_state(z, c):
    sd = ri.ppg2mel_state_dict(0)
    sd["decoder.stop_layer.linear_layer.weight"] = torch.from_numpy(z[c + "_stop_w"])
    sd["decoder.stop_layer.linear_layer.bias"] = torch.from_numpy(z[c + "_stop_b"])
    return sd


def case_masks(z, c):
    return (torch.from_numpy(np.unpackbits(z[c + "_mask1"], axis=-1)).bool(),
            torch.from_numpy(np.unpackbits(z[c + "_mask2"], axis=-1)).bool())


def model_for(sd):
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2

    m = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    m.load_state_dict(sd)
    m.eval()
    return m


@pytest.fixture(scope="module")
def model_c(golden):
    return model_for(case_state(golden, "c"))


def rel(got, ref):
    return po.rel_errors(got.cpu(), ref)


def pad_masks(m1, m2, S):
    """per-utterance masks padded to S steps (rows past the utterance's steps are never read)"""
    a = torch.zeros(S, 256, dtype=torch.bool)
    b = torch.zeros(S, 128, dtype=torch.bool)
    a[:m1.shape[0]], b[:m2.shape[0]] = m1[:S], m2[:S]
    return a, b


@pytest.mark.parametrize("case", CASES)
def test_golden_case(golden, case):
    z = golden
    m = model_for(case_state(z, case))
    T = z[case + "_ppg"].shape[0]
    masks = pad_masks(*case_masks(z, case), 2 * (T // 4))
    mel, post, align = m.inference(torch.from_numpy(z[case + "_ppg"])[None], torch.from_numpy(z[case + "_lf0_uv"])[None],
                                   torch.from_numpy(z[case + "_spk"])[None], dropout_masks=masks)
    assert mel.is_cuda and post.is_cuda and align.is_cuda
    assert align.shape == z[case + "_alignments"].shape, "step count differs from the reference"
    for name, got in (("mel", mel), ("mel_postnet", post), ("alignments", align)):
        e = rel(got, torch.from_numpy(z[f"{case}_{name}"]))
        print(f"golden {case} {name}: {e}")
        assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, (case, name, e)
    # the stop logits (scaled up to 53x in case c) stay well inside the fixture's 0.05 margin
    (_, _, _, stop), = m.inference_batch([(torch.from_numpy(z[case + "_ppg"]), torch.from_numpy(z[case + "_lf0_uv"]))],
                                         torch.from_numpy(z[case + "_spk"])[None], dropout_masks=[masks], return_stop=True)
    d = float((stop.cpu() - torch.from_numpy(z[case + "_stop"])).abs().max())
    print(f"golden {case} stop logits: max |diff| {d:.2e}")
    assert d <= 0.02, d


def random_utts(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    utts = [(torch.randn(T, 144, generator=g),
             torch.stack([torch.randn(T, generator=g), (torch.rand(T, generator=g) < 0.7).float()], 1)) for T in lengths]
    spk = torch.randn(len(lengths), 256, generator=g)
    masks = [(torch.rand(2 * (T // 4), 256, generator=g) < 0.5, torch.rand(2 * (T // 4), 128, generator=g) < 0.5)
             for T in lengths]
    return utts, spk, masks


def check_batch_vs_single(model, lengths, seed, oracle_rows=()):
    utts, spk, masks = random_utts(lengths, seed)
    batch = model.inference_batch(utts, spk, dropout_masks=masks)
    sd = case_state_cache[0]
    for i, ((ppg, lf0), res) in enumerate(zip(utts, batch)):
        one = model.inference(ppg[None], lf0[None], spk[i:i + 1], dropout_masks=masks[i])
        assert res[2].shape == one[2].shape, (i, lengths[i], "step count differs from the B = 1 call")
        for a, b in zip(res, one):
            assert torch.equal(a, b), (i, lengths[i], float((a - b).abs().max()))
        if i in oracle_rows:
            r = po.inference(sd, ppg, lf0, spk[i], masks=list(zip(*masks[i])))
            assert r["steps"] == res[2].shape[0]
            for name, got in (("mel", res[0]), ("mel_postnet", res[1]), ("alignments", res[2])):
                e = rel(got, r[name])
                assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, (i, name, e)
    return utts, spk, masks, batch


case_state_cache = []


@pytest.fixture(scope="module", autouse=True)
def _sd(golden):
    case_state_cache[:] = [case_state(golden, "c")]


def test_batch_mixed_lengths_equals_single_calls(model_c):
    check_batch_vs_single(model_c, [103, 262, 57, 400, 130, 8, 263], seed=11, oracle_rows=(0, 2, 5))


def test_batch_of_one_row(model_c):
    check_batch_vs_single(model_c, [97], seed=12, oracle_rows=(0,))


def test_batch_of_128_rows(model_c):
    lengths = torch.randint(20, 180, (128,), generator=torch.Generator().manual_seed(13)).tolist()
    check_batch_vs_single(model_c, lengths, seed=14, oracle_rows=(0, 77))


def test_batch_split_above_128_rows(model_c):
    lengths = torch.randint(8, 40, (130,), generator=torch.Generator().manual_seed(15)).tolist()
    utts, spk, masks = random_utts(lengths, 16)
    out = model_c.inference_batch(utts, spk, dropout_masks=masks)
    for i in (0, 129):
        one = model_c.inference(utts[i][0][None], utts[i][1][None], spk[i:i + 1], dropout_masks=masks[i])
        assert all(torch.equal(a, b) for a, b in zip(out[i], one))


def test_padding_frames_do_not_leak(model_c):
    lengths = [150, 61]
    utts, spk, masks = random_utts(lengths, 17)
    clean = model_c.inference_batch(utts, spk, dropout_masks=masks)
    from mockingbird_b200 import ppg2mel

    # the short row padded with large random values instead of zeros: drive _run directly with that padding
    dev = model_c._device
    T = max(lengths)
    g = torch.Generator().manual_seed(18)
    ppg = (torch.randn(2, T, 144, generator=g) * 1e3)
    lf0 = (torch.randn(2, T, 2, generator=g) * 1e3)
    for r, (p, l) in enumerate(utts):
        ppg[r, :lengths[r]], lf0[r, :lengths[r]] = p, l
    S = 2 * (T // 4)
    m1 = torch.zeros(S, 2, 256, dtype=torch.uint8)
    m2 = torch.zeros(S, 2, 128, dtype=torch.uint8)
    for r in range(2):
        s_r = masks[r][0].shape[0]
        m1[:s_r, r], m2[:s_r, r] = masks[r][0].to(torch.uint8), masks[r][1].to(torch.uint8)
        m1[s_r:, r], m2[s_r:, r] = 1, 1
    out = model_c._run(ppg.to(dev), lf0.to(dev), spk.to(dev).contiguous(), lengths, (m1, m2))
    assert ppg2mel.MAX_ROWS == 128
    for r in range(2):
        for a, b in zip(out[r], clean[r]):
            assert torch.equal(a, b), r


def test_device_dropout_seeded(model_c):
    utts, spk, _ = random_utts([90], 19)
    ppg, lf0 = utts[0]
    a = model_c.inference(ppg[None], lf0[None], spk, seed=5)
    b = model_c.inference(ppg[None], lf0[None], spk, seed=5)
    c = model_c.inference(ppg[None], lf0[None], spk, seed=6)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[0][:min(len(a[0]), len(c[0]))], c[0][:min(len(a[0]), len(c[0]))])
    S = 2 * (90 // 4)
    m1 = torch.stack([_philox_keep(5, s, 0, range(256), 1) for s in range(S)])
    m2 = torch.stack([_philox_keep(5, s, 0, range(128), 2) for s in range(S)])
    frac = float(torch.cat([m1.flatten(), m2.flatten()]).float().mean())
    assert 0.47 < frac < 0.53, frac
    r = po.inference(case_state_cache[0], ppg, lf0, spk[0], masks=list(zip(m1, m2)))
    assert r["steps"] == a[2].shape[0]
    e = rel(a[0], r["mel"])
    assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, e


def test_load_model_from_yaml_and_checkpoint(tmp_path, golden, model_c):
    import yaml

    from mockingbird_b200.ppg2mel import load_model

    (tmp_path / "ppg2mel.yaml").write_text(yaml.safe_dump({"model": dict(ri.PPG2MEL_CONFIG)}))
    torch.save({"model": case_state(golden, "c")}, tmp_path / "best_loss_step_0.pth")
    m = load_model(tmp_path / "best_loss_step_0.pth")
    utts, spk, masks = random_utts([120], 20)
    args = (utts[0][0][None], utts[0][1][None], spk)
    got = m.inference(*args, dropout_masks=masks[0])
    ref = model_c.inference(*args, dropout_masks=masks[0])
    assert all(torch.equal(x, y) for x, y in zip(got, ref))


def test_chain_into_hifigan(golden, model_c):
    import gan_oracle as go
    from mockingbird_b200.vocoder.hifigan.models import Generator

    cfg = ri.HIFIGAN_CONFIG_16K
    gsd = ri.hifigan_state_dict(cfg, 0)
    gen = Generator(cfg, precision="fp32").cuda()
    gen.load_state_dict(gsd)
    gen.eval()
    gen.remove_weight_norm()
    utts, spk, masks = random_utts([140], 21)
    ppg, lf0 = utts[0]
    _, post, _ = model_c.inference(ppg[None], lf0[None], spk, dropout_masks=masks[0])
    wav = gen(post.t()[None].contiguous()).cpu()
    r = po.inference(case_state_cache[0], ppg, lf0, spk[0], masks=list(zip(*masks[0])))
    with torch.no_grad():
        ref = go.hifigan_forward(gsd, cfg, r["mel_postnet"].t()[None])
    e = go.rel_errors(wav, ref)
    print(f"ppg2mel -> hifigan: {e}")
    assert e["max_rel"] <= TOL and e["rms_rel"] <= TOL, e


def test_bad_inputs_rejected(model_c):
    ppg, lf0, spk = torch.randn(1, 40, 144), torch.randn(1, 40, 2), torch.randn(1, 256)
    with pytest.raises(ValueError, match="frames"):
        model_c.inference(ppg, lf0[:, :39], spk)
    with pytest.raises(ValueError):
        model_c.inference(ppg[..., :100], lf0, spk)
    with pytest.raises(ValueError):
        model_c.inference(ppg, lf0[..., :1], spk)
    with pytest.raises(ValueError):
        model_c.inference(ppg, lf0, spk[:, :128])
    with pytest.raises(ValueError, match="B = 1"):
        model_c.inference(ppg.expand(2, -1, -1), lf0.expand(2, -1, -1), spk.expand(2, -1))
    with pytest.raises(ValueError):
        model_c.inference(ppg[:, :3], lf0[:, :3], spk)
    with pytest.raises(ValueError):
        model_c.inference(ppg, lf0, None)
