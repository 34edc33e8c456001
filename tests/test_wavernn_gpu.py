"""GPU parity tests of the WaveRNN path (through the drop-in surface -> C ABI).

  rung (i)   kernel == CPU twin, free running, bit-exact integer samples and bit-exact logits
  rung (iii) kernel under torch.manual_seed == the reference's golden samples / waveform
"""
import numpy as np
import pytest
import torch

import golden_io
import ref_init as ri
import wavernn_oracle as wo

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sd():
    return ri.wavernn_state_dict(0, randomize_bn=True)


@pytest.fixture(scope="module")
def model(sd):
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    return rnn_vocoder.load_state(sd)


@pytest.fixture(scope="module")
def twin(sd):
    return wo.Twin({k: v.numpy() for k, v in sd.items() if v.dtype == torch.float32})


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "wavernn_seed0.npz")


def test_kernel_equals_twin_injected_noise(model, twin):
    """ragged geometry: 7 frames, target 300 / overlap 40 -> 4 folds x 380 steps, last fold runs past
    the end of the conditioning (zero padding)"""
    mel = torch.rand(1, 80, 7, generator=torch.Generator().manual_seed(11)) * 2 - 1
    nf, starts = wo.fold_geometry(7 * 200, 300, 40)
    steps = 380
    noise = torch.empty(steps, nf, 512).exponential_(1, generator=torch.Generator().manual_seed(5))
    idx = model.generate_indices(mel, True, 300, 40, None, noise=noise)
    aux, melup = twin.condition(mel[0].numpy())
    ref = twin.generate(aux, melup, starts, steps, noise.numpy())
    assert idx.shape == ref.shape == (nf, steps)
    assert np.array_equal(idx, ref), f"first mismatch at {np.argwhere(idx != ref)[:3]}"


def test_kernel_equals_twin_device_rng(model, twin):
    mel = torch.rand(1, 80, 3, generator=torch.Generator().manual_seed(12)) * 2 - 1
    model.rng, model.seed = "device", 99
    try:
        idx = model.generate_indices(mel, False, 8000, 400, None)
    finally:
        model.rng = "torch"
    aux, melup = twin.condition(mel[0].numpy())
    ref = twin.generate(aux, melup, [0], 600, None, seed=99)
    assert np.array_equal(idx, ref)


def test_reference_golden_unbatched(model, gold):
    """BASELINE.json configs[0]-shaped: batched=False under torch.manual_seed(1234) reproduces the
    reference's integer samples and float64 waveform"""
    torch.manual_seed(1234)
    wav = model.generate(torch.from_numpy(gold["mel1"]), False, 8000, 400, True, progress_callback=lambda *a: None)
    assert wav.dtype == np.float64 and wav.shape == gold["wav1"].shape
    assert np.abs(wav - gold["wav1"]).max() <= 1e-12
    assert model.training  # generate() leaves the module in train mode like the reference (:255)


def test_reference_golden_batched(model, gold):
    """configs[2]-shaped: fold / cross-fade path (6 folds x 1200 steps)"""
    calls = []
    torch.manual_seed(1234)
    wav = model.generate(torch.from_numpy(gold["mel2"]), True, 1000, 100, True,
                         progress_callback=lambda i, n, b, r: calls.append((i, n, b)))
    assert np.abs(wav - gold["wav2"]).max() <= 1e-12
    assert calls[0] == (0, 1200, 6) and calls[-1] == (1100, 1200, 6) and len(calls) == 12


def test_more_than_one_row_block(model, twin):
    """70 folds -> two 64-row blocks inside the kernel"""
    mel = torch.rand(1, 80, 40, generator=torch.Generator().manual_seed(13)) * 2 - 1
    nf, starts = wo.fold_geometry(40 * 200, 100, 12)
    assert nf > 64
    steps = 124
    noise = torch.empty(steps, nf, 512).exponential_(1, generator=torch.Generator().manual_seed(6))
    idx = model.generate_indices(mel, True, 100, 12, None, noise=noise)
    aux, melup = twin.condition(mel[0].numpy())
    ref = twin.generate(aux, melup, starts, steps, noise.numpy())
    assert np.array_equal(idx, ref)


def test_inference_module_protocol(tmp_path, sd, gold):
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    rnn_vocoder._model = None
    with pytest.raises(Exception, match="Please load Wave-RNN"):
        rnn_vocoder.infer_waveform(np.zeros((80, 30), np.float32))
    torch.save({"model_state": sd}, tmp_path / "wavernn.pt")
    rnn_vocoder.load_model(tmp_path / "wavernn.pt", "ignored_config", verbose=False)
    assert rnn_vocoder.is_loaded()
    torch.manual_seed(1234)
    wav, sr = rnn_vocoder.infer_waveform(gold["mel2"][0] * 4.0, batched=True, target=1000, overlap=100,
                                         progress_callback=lambda *a: None)
    assert sr == 16000
    assert np.abs(wav - gold["wav2"]).max() <= 1e-12


@pytest.mark.parametrize("rng", ["torch", "device"])
def test_fold_rows_independent_of_sharding(model, rng):
    """SURVEY.md 8e row 2: the folds of one utterance are independent rows; running them as [0,3) + [3,8) (what two
    GPUs would do) gives exactly the rows of the single call, and leaves the torch generator in the same state"""
    mel = torch.rand(1, 80, 13, generator=torch.Generator().manual_seed(21)) * 2 - 1
    model.rng, model.seed = rng, 31
    try:
        torch.manual_seed(55)
        full = model.generate_indices(mel, True, 300, 35, None)
        tail = torch.rand(3)
        parts = []
        for lo, hi in ((0, 3), (3, 8), (8, 8)):
            torch.manual_seed(55)
            parts.append(model.generate_indices(mel, True, 300, 35, None, rows=(lo, hi)))
            assert torch.equal(torch.rand(3), tail) or rng == "device"
    finally:
        model.rng = "torch"
    assert full.shape == (8, 370) and parts[2].shape == (0, 370)
    assert np.array_equal(np.concatenate(parts), full)


def test_device_postprocess_matches_reference(model, gold, golden_dir):
    """mb_wavernn_postprocess (float64 kernels: unfold + cross-fade, mu-law, parallel de-emphasis, fade) on the reference's own
    integer samples == the reference's float64 waveform, <= 1e-12 (the host numpy path holds the same bound)"""
    import json

    w1 = model.postprocess_device(torch.from_numpy(gold["idx1"]).cuda(), 27, False, 8000, 400, True)
    assert w1.dtype == np.float64 and w1.shape == gold["wav1"].shape and np.abs(w1 - gold["wav1"]).max() <= 1e-12
    w2 = model.postprocess_device(torch.from_numpy(gold["idx2"]).cuda(), 30, True, 1000, 100, True)
    assert w2.shape == gold["wav2"].shape and np.abs(w2 - gold["wav2"]).max() <= 1e-12
    z = golden_io.load(golden_dir / "wavernn_cfg3.npz")
    w3 = model.postprocess_device(torch.from_numpy(z["idx"]).cuda(), 2400, True, 8000, 400, True)
    st = int(json.loads(str(z["meta"]))["wav_stride"])
    assert len(w3) == int(z["wav_len"])
    assert np.abs(w3[::st] - z["wav_strided"]).max() <= 1e-12
    assert np.abs(w3[:4096] - z["wav_head"]).max() <= 1e-12 and np.abs(w3[-8192:] - z["wav_tail"]).max() <= 1e-12
    # and against the host restatement on every sample
    host = model.postprocess(z["idx"], 2400, True, 8000, 400, True)
    assert np.abs(w3 - host).max() <= 1e-13
