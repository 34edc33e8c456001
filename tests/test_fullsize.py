"""Parity at the BASELINE.json configuration sizes against fixtures generated from the LIVE reference by
oracle/make_golden_full.py (cfg 1: 16 000 unbatched draws; cfg 3: 58 folds x 8 800 draws; cfg 4: Tacotron B = 64, <= 120
chars, 400 frames; Fre-GAN on the cfg-2 shape).  CPU tests pin the oracle at these sizes; GPU tests are the parity tests
proper (through the drop-in surface -> C ABI).  Integer samples: identical; float: <= 1e-3 relative (north_star)."""
import json

import numpy as np
import pytest
import torch

import golden_io
import ref_init as ri
import wavernn_oracle as wo


def _noise_rows(seed, B, steps, rows):
    """the Exp(1) stream of WaveRNN.generate (SURVEY.md fact 5), keeping only some fold rows"""
    torch.manual_seed(seed)
    torch.nn.GRUCell(512, 512)
    torch.nn.GRUCell(544, 512)
    out = torch.empty(steps, len(rows), 512)
    buf = torch.empty(B, 512)
    for i in range(steps):
        buf.exponential_(1)
        out[i] = buf[rows]
    return out


def _first_divergence(idx, ref):
    bad = np.argwhere(idx != ref)
    if len(bad) == 0:
        return None
    step = int(bad[:, 1].min())
    rows = sorted(set(int(r) for r, s in bad if s == step))
    return {"first_step": step, "rows_at_first_step": rows, "n_diff": int(len(bad)),
            "rows_diverged": int(len(set(bad[:, 0])))}


MEL1 = lambda: torch.rand(1, 80, 80, generator=torch.Generator().manual_seed(1)) * 2 - 1      # noqa: E731
MEL3 = lambda: torch.rand(1, 80, 2400, generator=torch.Generator().manual_seed(3)) * 2 - 1    # noqa: E731


@pytest.fixture(scope="module")
def wsd():
    return ri.wavernn_state_dict(0, randomize_bn=True)


@pytest.fixture(scope="module")
def twin(wsd):
    return wo.Twin({k: v.numpy() for k, v in wsd.items() if v.dtype == torch.float32})


# ---------------------------------------------------------------- CPU: oracle pinned at full size
def test_twin_cfg1_all_16000_draws(twin, golden_dir):
    """BASELINE.json configs[0]: free-running twin == reference on every one of the 16 000 draws"""
    z = np.load(golden_dir / "wavernn_cfg1.npz")
    aux, melup = twin.condition(MEL1()[0].numpy())
    noise = ri.wavernn_noise(1234, 1, 16000).numpy()
    idx = twin.generate(aux, melup, [0], 16000, noise)
    assert _first_divergence(idx, z["idx"]) is None
    wav = wo.postprocess(idx, 80, False, 8000, 400, ri.WAVERNN_HP)
    assert np.abs(wav - z["wav"]).max() <= 1e-12


def test_twin_cfg3_three_folds_all_8800_draws(twin, golden_dir):
    """configs[2]: folds 0, 29 and 57 (the last one runs past the end of the conditioning) free running for all
    8 800 steps == the reference; the post-processing restatement reproduces the reference waveform from the
    golden integers"""
    z = golden_io.load(golden_dir / "wavernn_cfg3.npz")
    nf, starts = wo.fold_geometry(2400 * 200, 8000, 400)
    assert nf == 58 and z["idx"].shape == (58, 8800)
    rows = [0, 29, 57]
    aux, melup = twin.condition(MEL3()[0].numpy())
    noise = _noise_rows(1234, 58, 8800, rows).numpy()
    idx = twin.generate(aux, melup, starts[rows], 8800, noise)
    assert _first_divergence(idx, z["idx"][rows]) is None
    wav = wo.postprocess(z["idx"], 2400, True, 8000, 400, ri.WAVERNN_HP)
    assert len(wav) == int(z["wav_len"])
    st = int(json.loads(str(z["meta"]))["wav_stride"])
    assert np.abs(wav[::st] - z["wav_strided"]).max() <= 1e-12
    assert np.abs(wav[:4096] - z["wav_head"]).max() <= 1e-12 and np.abs(wav[-8192:] - z["wav_tail"]).max() <= 1e-12


def test_tacotron_oracle_cfg4_rows(golden_dir):
    """configs[3]: the torch-CPU oracle with the captured masks == the reference on the stored rows (cheap slice:
    the four stored utterances as their own batch; rows of a batch are independent in eval mode)"""
    import tacotron_oracle as to

    z = golden_io.load(golden_dir / "tacotron_cfg4.npz")
    rows = [int(r) for r in z["rows"]]
    chars = torch.from_numpy(z["chars"].astype(np.int64))
    emb = torch.from_numpy(z["emb"])
    enc = torch.from_numpy(np.unpackbits(z["enc_masks"], axis=-1)).bool()
    dec = torch.from_numpy(np.unpackbits(z["dec_masks"], axis=-1)).bool()
    steps = 40  # first 40 frames = 20 decoder iterations
    masks = [enc[0][rows], enc[1][rows]] + [dec[i][rows] for i in range(steps)]
    sd = ri.tacotron_state_dict(0, r=2, randomize_bn=True)
    mel, lin, attn = to.generate(sd, chars[rows], emb[rows], steps, -1, 10, masks, r=2)
    ref = torch.from_numpy(z["mel"])[:, :, :steps]
    assert float((mel - ref).abs().max() / ref.abs().max()) <= 1e-5
    ref_a = torch.from_numpy(z["attn"])[:, :steps // 2]
    assert float((attn - ref_a).abs().max()) <= 1e-5


# ---------------------------------------------------------------- GPU: parity proper
@pytest.fixture(scope="module")
def wmodel(wsd):
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    return rnn_vocoder.load_state(wsd)


@pytest.mark.gpu
def test_gpu_wavernn_cfg1_identical(wmodel, golden_dir):
    z = np.load(golden_dir / "wavernn_cfg1.npz")
    torch.manual_seed(1234)
    idx = wmodel.generate_indices(MEL1(), False, 8000, 400, None)
    assert _first_divergence(idx, z["idx"]) is None
    torch.manual_seed(1234)
    wav = wmodel.generate(MEL1(), False, 8000, 400, True, progress_callback=lambda *a: None)
    assert wav.shape == z["wav"].shape and np.abs(wav - z["wav"]).max() <= 1e-12


@pytest.mark.gpu
def test_gpu_wavernn_cfg3_identical(wmodel, golden_dir):
    """all 58 x 8 800 = 510 400 draws integer-identical to the reference's CPU run under torch.manual_seed(1234);
    a mismatch reports the first diverging step and rows"""
    z = golden_io.load(golden_dir / "wavernn_cfg3.npz")
    torch.manual_seed(1234)
    idx = wmodel.generate_indices(MEL3(), True, 8000, 400, None)
    assert idx.shape == (58, 8800)
    assert _first_divergence(idx, z["idx"]) is None
    torch.manual_seed(1234)
    wav = wmodel.generate(MEL3(), True, 8000, 400, True, progress_callback=lambda *a: None)
    st = int(json.loads(str(z["meta"]))["wav_stride"])
    assert len(wav) == int(z["wav_len"])
    assert np.abs(wav[::st] - z["wav_strided"]).max() <= 1e-12
    assert np.abs(wav[:4096] - z["wav_head"]).max() <= 1e-12 and np.abs(wav[-8192:] - z["wav_tail"]).max() <= 1e-12
    assert abs(wav.sum() - float(z["wav_sum"][0])) <= 1e-7 and abs(np.abs(wav).sum() - float(z["wav_sum"][1])) <= 1e-7


@pytest.mark.gpu
def test_gpu_tacotron_cfg4(golden_dir):
    """B = 64, <= 120 chars, 400 frames = 200 recurrent steps through the 3-term-split LSTMs, injected reference masks:
    stored rows within 1e-3 (max-norm relative, asserted at 5e-4), every row's float64 sums, attention argmax path"""
    from mockingbird_b200.synthesizer.inference import Synthesizer

    z = golden_io.load(golden_dir / "tacotron_cfg4.npz")
    model = Synthesizer("unused.pt", verbose=False).load_state(ri.tacotron_state_dict(0, r=2, randomize_bn=True))
    chars = torch.from_numpy(z["chars"].astype(np.int64))
    emb = torch.from_numpy(z["emb"])
    enc = torch.from_numpy(np.unpackbits(z["enc_masks"], axis=-1))
    dec = np.unpackbits(z["dec_masks"], axis=-1)
    dec = torch.from_numpy(dec.reshape(-1, 2, dec.shape[-2], dec.shape[-1]))
    steps, style, mst, r = [int(v) for v in z["cfg"]]
    model.r = r
    mel, lin, attn = model.generate(chars, emb, steps=steps, style_idx=style, min_stop_token=mst, dropout_masks=(enc, dec))
    assert mel.shape == (64, 80, 400) and attn.shape == (64, 200, 120)
    rows = [int(v) for v in z["rows"]]
    mel, lin, attn = mel.cpu(), lin.cpu(), attn.cpu()
    TOL = 5e-4
    for got, key, scale in ((mel, "mel", float(z["mel_absmax"])), (lin, "linear", float(z["linear_absmax"])), (attn, "attn", 1.0)):
        ref = torch.from_numpy(z[key])
        err = float((got[rows] - ref).abs().max()) / scale
        assert err <= TOL, (key, err)
    # every row, through size-independent summaries of the reference output
    for got, key in ((mel, "mel"), (lin, "linear")):
        s = got.double().sum(dim=(1, 2)).numpy()
        a = got.double().abs().sum(dim=(1, 2)).numpy()
        assert np.max(np.abs(s - z[f"{key}_rowsum"]) / z[f"{key}_rowabs"]) <= TOL, key
        assert np.max(np.abs(a - z[f"{key}_rowabs"]) / z[f"{key}_rowabs"]) <= TOL, key
    agree = float((attn.argmax(dim=2).numpy() == z["attn_argmax"]).mean())
    assert agree >= 0.999, agree


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "f16tc"])
def test_gpu_fregan_cfg2_rows(golden_dir, precision):
    """Fre-GAN on the cfg-2 shape (32 x 256 frames): rows 0 and 31 against the reference, 1e-3 both metrics"""
    import gan_oracle as go
    from mockingbird_b200.vocoder.fregan.models import FreGAN

    z = np.load(golden_dir / "fregan_cfg2.npz")
    g = FreGAN(ri.FREGAN_CONFIG, precision=precision).cuda()
    g.load_state_dict(ri.fregan_state_dict(ri.FREGAN_CONFIG, 0))
    g.eval()
    g.remove_weight_norm()
    mel = torch.rand(32, 80, 256, generator=torch.Generator().manual_seed(2)) * 8 - 4
    wav = g(mel.cuda())
    assert wav.shape == (32, 1, 51200)
    pick = [int(i) for i in z["full_pick"]]
    e = go.rel_errors(wav[pick].cpu(), torch.from_numpy(z["wav_full"]))
    tol = 2e-5 if precision == "fp32" else 1e-3
    assert e["max_rel"] <= tol and e["rms_rel"] <= tol, e


def test_torch_oracle_prefix_matches_reference(wsd, golden_dir):
    """the torch-CPU restatement used as bench.py's WaveRNN CPU leg == the reference on a prefix of cfg 1 (400 draws)
    and of cfg 3 (58 folds x 40 steps) under the same seed"""
    import wavernn_torch_oracle as wt

    z1 = np.load(golden_dir / "wavernn_cfg1.npz")
    torch.manual_seed(1234)
    idx, _ = wt.generate_indices(wsd, MEL1(), False, 8000, 400, max_steps=400)
    assert np.array_equal(idx, z1["idx"][:, :400])
    z3 = golden_io.load(golden_dir / "wavernn_cfg3.npz")
    torch.manual_seed(1234)
    idx, _ = wt.generate_indices(wsd, MEL3(), True, 8000, 400, max_steps=40)
    assert np.array_equal(idx, z3["idx"][:, :40])
