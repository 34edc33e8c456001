"""CPU tests of the PPG extractor: the plain-torch restatement against the golden vectors and the live reference, the
seeded weights against the reference constructor, the restated quirks (legacy rel_shift, positional-table high-water
mark, var^(1/4) normalisation), and the C ABI's config checks and frame counts (host-only, no device)."""
import ctypes as C

import numpy as np
import pytest
import torch

import golden_io
import ppgx_oracle as po
import ref_init as ri
from mockingbird_b200 import _lib
from mockingbird_b200.ppg_extractor import build_model, pos_table

VARIANTS = dict(small=ri.PPGX_CONFIG_SMALL, **ri.PPGX_SMALL_VARIANTS)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return golden_io.load(golden_dir / "ppgx_seed0.npz")


def close(a, b, tol=1e-5):
    return float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max()))


def test_oracle_matches_golden(golden):
    z = golden
    out, taps = po.forward(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0), ri.PPGX_CONFIG, torch.from_numpy(z["a_wav"]),
                           taps=True)
    assert close(out, torch.from_numpy(z["a_out"]))
    for i, ref in zip(z["a_tap_index"], z["a_taps"]):
        assert close(taps[i], torch.from_numpy(ref)), i
    for name, cfg in VARIANTS.items():
        out = po.forward(ri.ppg_extractor_state_dict(cfg, 0), cfg, torch.from_numpy(z["v_wav"]))
        assert out.shape == z[f"v_{name}_out"].shape and close(out, torch.from_numpy(z[f"v_{name}_out"])), name


def test_fixture_shapes(golden):
    z = golden
    assert z["a_out"].shape == (301, 144) and z["b_out"].shape == (ri.ppgx_frames(ri.PPGX_CONFIG, len(z["b_wav"])), 144)
    assert (z["a_wav"][19200:21600] == 0).all()  # the run of exact zeros (log(1e-20) frames)
    assert int(z["long_pe_len"]) == ri.ppgx_frames(ri.PPGX_CONFIG_SMALL, int(z["long_n"])) > 5000
    assert int(z["short_pe_len"]) == int(z["long_pe_len"])


@pytest.mark.reference
def test_restatement_matches_live_reference():
    import ppgx_harness as ph

    if not ph.reference_available():
        pytest.skip("reference tree not available")
    g = np.random.RandomState(9)
    for cfg in (ri.PPGX_CONFIG_SMALL, ri.PPGX_SMALL_VARIANTS["abs_pos"], ri.PPGX_SMALL_VARIANTS["no_vars"],
                ri.PPGX_SMALL_VARIANTS["vars_only"], ri.PPGX_SMALL_VARIANTS["fe_defaults"]):
        m = ph.build_ppg_extractor(cfg, 1)
        sd = ri.ppg_extractor_state_dict(cfg, 1)
        m.load_state_dict(sd)
        wav = (0.2 * g.randn(12640)).astype(np.float32)
        with torch.no_grad():
            ref = m(torch.from_numpy(wav)[None], torch.LongTensor([len(wav)]))[0]
        assert torch.equal(po.forward(sd, cfg, torch.from_numpy(wav)), ref)


@pytest.mark.reference
def test_state_dict_bit_identical_to_reference_constructor():
    import ppgx_harness as ph

    if not ph.reference_available():
        pytest.skip("reference tree not available")
    for cfg in [ri.PPGX_CONFIG] + list(VARIANTS.values()):
        ref = ph.build_ppg_extractor(cfg, 0).state_dict()
        sd = ri.ppg_extractor_state_dict(cfg, 0, randomize_bn=False)
        assert list(ref) == list(sd)
        for k in ref:
            assert ref[k].shape == sd[k].shape and torch.equal(ref[k], sd[k]), k
    ref = ph.build_ppg_extractor(ri.PPGX_CONFIG, 0).state_dict()
    n = sum(v.numel() for k, v in ref.items() if v.dtype.is_floating_point and "running" not in k and "melmat" not in k)
    assert n == 10_252_512


def test_rel_shift_closed_form():
    g = torch.Generator().manual_seed(0)
    for T in (1, 2, 5, 9):
        bd = torch.randn(3, T, T, generator=g)
        assert torch.equal(po.rel_shift(bd), po.rel_shift_closed_form(bd))


def test_pe_len_rule():
    """row k of the rel_pos table encodes position pe_len - 1 - k: query i / key j see pe_len - T + i - j, which depends on
    T and on the instance's longest input"""
    D = 8
    for pe_len in (5000, 5011):
        tab = po.pos_table(D, pe_len, reverse=True)
        pos = torch.tensor([float(pe_len - 1 - k) for k in range(12)])
        div = torch.exp(torch.arange(0, D, 2).float() * -(np.log(10000.0) / D))
        assert torch.allclose(tab[:12, 0::2], torch.sin(pos[:, None] * div), atol=1e-4)
        assert torch.equal(pos_table(D, pe_len, True), tab)
    assert torch.equal(pos_table(D, 5000, False), po.pos_table(D, 5000, False))
    assert not torch.equal(po.pos_table(D, 5000, True)[:10], po.pos_table(D, 5011, True)[:10])


def test_mvn_divides_by_var_fourth_root():
    cfg = ri.PPGX_CONFIG_SMALL
    sd = ri.ppg_extractor_state_dict(cfg, 0)
    wav = torch.from_numpy((0.1 * np.random.RandomState(2).randn(8000)).astype(np.float32))
    x = po.features(sd, cfg, wav)
    cfg_raw = ri._ppgx_variant(cfg, normalize=dict(norm_means=False, norm_vars=False))
    raw = po.features(sd, cfg_raw, wav)
    c = raw - raw.mean(0)
    assert torch.allclose(x, c / c.pow(2).mean(0).pow(0.25), rtol=1e-4, atol=1e-5)


def test_num_frames_matches_restatement():
    for cfg in [ri.PPGX_CONFIG] + list(VARIANTS.values()):
        m = build_model(cfg)
        for n in (201, 1000, 15877, 48000, 160 * 5010):
            assert m.num_frames(n) == ri.ppgx_frames(cfg, n) == po.num_frames(cfg, n)


def test_handle_on_cpu():
    m = build_model(ri.PPGX_CONFIG)
    L = _lib.lib()
    assert L.mb_ppgx_arena_bytes(m._handle) >= 10_252_512 * 4
    assert L.mb_ppgx_workspace_bytes(m._handle, 2, 48000) > 0
    assert L.mb_ppgx_workspace_bytes(m._handle, 2, 200) == 0  # reflect padding needs more than n_fft / 2 samples
    assert L.mb_ppgx_workspace_bytes(m._handle, 129, 48000) == 0
    assert L.mb_ppgx_finalize(m._handle, None) == 2  # no arena / weights yet


def _enc(**over):
    return ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, **over)


@pytest.mark.parametrize("cfg,what", [
    (_enc(input_layer="linear"), b"input_layer"),
    (_enc(pos_enc_layer_type="scaled_abs_pos", selfattention_layer_type="selfattn"), b"scaled_abs_pos"),
    (_enc(concat_after=True), b"concat_after"),
    (_enc(normalize_before=False), b"normalize_before"),
    (_enc(positionwise_layer_type="conv1d"), b"positionwise_layer_type"),
    (_enc(positionwise_layer_type="conv1d-linear"), b"positionwise_layer_type"),
    (ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, frontend=dict(kaldi_padding_mode=True)), b"kaldi_padding_mode"),
    (ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, frontend=dict(downsample_rate=2)), b"downsample_rate"),
    (_enc(attention_dim=32, attention_heads=3), b"not divisible"),
    (_enc(pos_enc_layer_type="abs_pos"), b"rel_selfattn"),
])
def test_unsupported_config_rejected(cfg, what):
    L = _lib.lib()
    with pytest.raises(_lib.MbError) as e:
        build_model(cfg)
    assert "error 1" in str(e.value)
    assert what in L.mb_last_error()


def test_module_rejects_cpu_device():
    m = build_model(ri.PPGX_CONFIG_SMALL)
    with pytest.raises(_lib.MbError):
        m.to("cpu")


@pytest.mark.reference
def test_frontend_defaults_match_reference():
    """a frontend_conf without the STFT keys gets DefaultFrontend's own defaults (n_fft 1024, win_length 800, hop 160)"""
    import ppgx_harness as ph

    if not ph.reference_available():
        pytest.skip("reference tree not available")
    cfg = ri.PPGX_SMALL_VARIANTS["fe_defaults"]
    assert not {"n_fft", "win_length", "hop_length"} & set(cfg["frontend_conf"])
    ref = ph.build_ppg_extractor(cfg, 0)
    st = ref.frontend.stft
    assert (st.n_fft, st.win_length, st.hop_length) == (1024, 800, 160) == po.stft_params(cfg)
    m = build_model(cfg)
    assert (m.cfg.n_fft, m.cfg.win_length, m.cfg.hop_length) == (1024, 800, 160)
    assert tuple(m._default_melmat.shape) == tuple(ref.state_dict()["frontend.logmel.melmat"].shape) == (513, 80)
    assert torch.equal(m._default_melmat, ref.state_dict()["frontend.logmel.melmat"])
    for n in (12640, 16000, 48000):
        with torch.no_grad():
            T = ref(torch.zeros(1, n) + 0.01 * torch.randn(1, n), torch.LongTensor([n])).shape[1]
        assert m.num_frames(n) == T == ri.ppgx_frames(cfg, n) == po.num_frames(cfg, n)


def _fe(**over):
    return ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, frontend=over)


@pytest.mark.parametrize("cfg,what", [
    (_fe(center=False), "center"),
    (_fe(pad_mode="constant"), "pad_mode"),
    (_fe(normalized=True), "normalized"),
    (_fe(onesided=False), "onesided"),
    (_fe(htk=True), "htk"),
    (_fe(norm=2), "norm"),
    (_fe(frontend_conf=dict(use_wpe=True)), "frontend_conf"),
    (_fe(n_mels=40), "n_mels"),
    (_fe(window="hann"), "unexpected keys"),
    (dict(frontend_conf={k: v for k, v in ri.PPGX_CONFIG_SMALL["frontend_conf"].items() if k != "fs"},
          normalize_conf=ri.PPGX_CONFIG_SMALL["normalize_conf"], encoder_conf=ri.PPGX_CONFIG_SMALL["encoder_conf"]), "fs"),
    (ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, normalize=dict(eps=1e-10)), "eps"),
    (_enc(dropout=0.1), "unexpected keys"),
])
def test_unsupported_frontend_options_rejected(cfg, what):
    with pytest.raises(_lib.MbError, match=what):
        build_model(cfg)


def test_frontend_norm_slaney_is_the_area_rule():
    from mockingbird_b200.synthesizer.audio_host import mel_basis

    m = build_model(_fe(norm="slaney"))
    assert torch.allclose(m._default_melmat, torch.from_numpy(mel_basis(16000, 400, 80, 0.0, 8000.0).T), rtol=1e-6, atol=0)
