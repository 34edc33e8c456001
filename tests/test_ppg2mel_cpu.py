"""CPU tests of the voice-conversion mel decoder (ppg2mel): the oracle against the golden vectors from the live
reference, the seeded weights against the reference constructor, the fixture's stop-logit margins, and the C ABI's
config checks (host-only, no device)."""
import ctypes as C

import numpy as np
import pytest
import torch

import golden_io
import ppg2mel_oracle as po
import ref_init as ri
from mockingbird_b200 import _lib

CASES = ("a", "b", "c")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return golden_io.load(golden_dir / "ppg2mel_seed0.npz")


def case_state(z, c):
    sd = ri.ppg2mel_state_dict(0)
    sd["decoder.stop_layer.linear_layer.weight"] = torch.from_numpy(z[c + "_stop_w"])
    sd["decoder.stop_layer.linear_layer.bias"] = torch.from_numpy(z[c + "_stop_b"])
    return sd


def case_masks(z, c):
    m1 = torch.from_numpy(np.unpackbits(z[c + "_mask1"], axis=-1)).bool()
    m2 = torch.from_numpy(np.unpackbits(z[c + "_mask2"], axis=-1)).bool()
    return m1, m2


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_golden(golden, case):
    z = golden
    m1, m2 = case_masks(z, case)
    r = po.inference(case_state(z, case), torch.from_numpy(z[case + "_ppg"]), torch.from_numpy(z[case + "_lf0_uv"]),
                     torch.from_numpy(z[case + "_spk"]), masks=list(zip(m1, m2)))
    assert r["steps"] == z[case + "_alignments"].shape[0]
    for k in ("mel", "mel_postnet", "alignments", "stop"):
        ref = torch.from_numpy(z[f"{case}_{k}"])
        assert r[k].shape == ref.shape, k
        assert float((r[k] - ref).abs().max()) <= 1e-6 * max(1.0, float(ref.abs().max())), k


def test_fixture_covers_the_termination_paths(golden):
    z = golden
    kinds = {}
    for c in CASES:
        T = z[c + "_ppg"].shape[0]
        n, te = z[c + "_alignments"].shape
        assert te == (T // 2) // 2 and z[c + "_mel"].shape == (2 * n, 80) and z[c + "_mel_postnet"].shape == (2 * n, 80)
        mx, mn = 2 * te, 2 * te - 5
        stop = z[c + "_stop"]
        assert stop.shape == (n,)
        # every decisive step (n >= min_decoder_step) is at least 0.05 away from the threshold
        assert (np.abs(stop[mn - 1:n]) >= 0.05).all()
        assert (stop[mn - 1:n - 1] < 0).all()
        if n == mx and stop[n - 1] < 0:
            kinds[c] = "max"
        elif n == mn:
            kinds[c] = "min"
        else:
            assert mn < n < mx and stop[n - 1] > 0
            kinds[c] = "sigmoid"
        assert z[c + "_mask1"].shape == (n, 32) and z[c + "_mask2"].shape == (n, 16)
    assert sorted(kinds.values()) == ["max", "min", "sigmoid"]
    assert any(z[c + "_ppg"].shape[0] % 4 for c in CASES)


@pytest.mark.reference
def test_state_dict_bit_identical_to_reference_constructor():
    import ref_harness as rh

    if not rh.reference_available():
        pytest.skip("reference tree not available")
    rh.install()
    from models.ppg2mel import MelDecoderMOLv2

    torch.manual_seed(0)
    ref = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).state_dict()
    sd = ri.ppg2mel_state_dict(0, randomize_bn=False)
    assert list(ref) == list(sd)
    for k in ref:
        assert ref[k].shape == sd[k].shape and torch.equal(ref[k], sd[k]), k
    n = sum(v.numel() for k, v in ref.items() if v.dtype.is_floating_point and "running" not in k)
    assert n == 10_396_576


def _cfg(**over):
    cfg = _lib.Ppg2MelConfig()
    cfg.bottle_neck_feature_dim, cfg.spk_embed_dim, cfg.encoder_dim = 144, 256, 256
    cfg.encoder_downsample_rates[0] = cfg.encoder_downsample_rates[1] = 2
    cfg.attention_rnn_dim = cfg.decoder_rnn_dim = 512
    cfg.num_decoder_rnn_layer, cfg.concat_context_to_last = 1, 1
    cfg.prenet_dims[0], cfg.prenet_dims[1] = 256, 128
    cfg.num_mixtures, cfg.frames_per_step, cfg.num_mels = 5, 2, 80
    for k, v in over.items():
        if isinstance(v, tuple):
            getattr(cfg, k)[v[0]] = v[1]
        else:
            setattr(cfg, k, v)
    return cfg


def test_default_config_handle_on_cpu():
    lib = _lib.lib()
    h = C.c_void_p()
    _lib.check(lib.mb_ppg2mel_create(C.byref(_cfg()), C.byref(h)))
    try:
        assert lib.mb_ppg2mel_arena_bytes(h) >= 10_396_576 * 4 - 128 * 256 * 4 - 256 * 80 * 4
        assert lib.mb_ppg2mel_workspace_bytes(h, 2, 100) > 0
        assert lib.mb_ppg2mel_workspace_bytes(h, 2, 3) == 0
        assert lib.mb_ppg2mel_finalize(h, None) == 2  # no arena / weights yet
    finally:
        lib.mb_ppg2mel_destroy(h)


@pytest.mark.parametrize("field,value", [
    ("encoder_dim", 128), ("encoder_downsample_rates", (0, 3)), ("encoder_downsample_rates", (1, 4)),
    ("attention_rnn_dim", 1024), ("decoder_rnn_dim", 256), ("num_decoder_rnn_layer", 2), ("concat_context_to_last", 0),
    ("prenet_dims", (0, 128)), ("prenet_dims", (1, 256)), ("num_mixtures", 4), ("frames_per_step", 1),
    ("num_mels", 40), ("bottle_neck_feature_dim", 0), ("spk_embed_dim", 4096)])
def test_unsupported_config_rejected(field, value):
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.mb_ppg2mel_create(C.byref(_cfg(**{field: value})), C.byref(h)) == 1
    assert field.encode() in lib.mb_last_error()


def test_module_rejects_bad_config_and_cpu_device():
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2

    with pytest.raises(_lib.MbError):
        MelDecoderMOLv2(num_speakers=1, spk_embed_dim=256, bottle_neck_feature_dim=144, num_mixtures=8)
    m = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG)
    with pytest.raises(_lib.MbError):
        m.to("cpu")
