"""GPU tests of the multi-utterance WaveRNN sample loop (WaveRNN.generate_many, mb_wavernn_condition_multi /
mb_wavernn_generate_multi[_mol], k_sample_loop<MOL>): every utterance of a batch is bit for bit what the
single-utterance call returns for it alone - conditioning tables, ragged lengths, per-utterance noise, RAW and MOL."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

import ref_init as ri
import wavernn_mol_oracle as mo
import wavernn_oracle as wo

pytestmark = pytest.mark.gpu

MODES = ["RAW", "MOL"]
TOL_MOL = 1e-3  # the MOL sampler's bound against the reference (tests/test_wavernn_mol_gpu.py)


@pytest.fixture(scope="module")
def golds(golden_dir):
    return {"RAW": np.load(golden_dir / "wavernn_seed0.npz"), "MOL": np.load(golden_dir / "wavernn_mol_seed0.npz")}


@pytest.fixture(scope="module")
def sds(golds):
    mol = ri.wavernn_state_dict(0, randomize_bn=True, mode="MOL")
    mol["fc3.bias"] = mol["fc3.bias"].clone()
    mol["fc3.bias"][20:30] += json.loads(str(golds["MOL"]["meta"]))["log_scale_shift"]
    return {"RAW": ri.wavernn_state_dict(0, randomize_bn=True), "MOL": mol}


@pytest.fixture(scope="module")
def models(sds):
    from mockingbird_b200.vocoder.wavernn import hparams as hp
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    out = {}
    old = hp.voc_mode
    try:
        for mode in MODES:
            hp.voc_mode = mode
            out[mode] = rnn_vocoder.load_state(sds[mode])
    finally:
        hp.voc_mode = old
    rnn_vocoder._model = None
    return out


def _mels(lengths, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(1, 80, T, generator=g) * 2 - 1 for T in lengths]


def _noise(mode, steps, B, seed):
    g = torch.Generator().manual_seed(seed)
    if mode == "RAW":
        return torch.empty(steps, B, 512).exponential_(1, generator=g)
    return torch.empty(steps, 11 * B).uniform_(1e-5, 1.0 - 1e-5, generator=g)


def _single(model, mel, batched, target, overlap, noise=None):
    run = model.generate_samples if model.mode == "MOL" else model.generate_indices
    return run(mel, batched, target, overlap, None, noise=noise)


def _same(many, singles):
    for u, (a, b) in enumerate(zip(many, singles)):
        a = a.cpu().numpy()
        assert a.shape == b.shape and a.dtype == b.dtype, (u, a.shape, b.shape)
        assert np.array_equal(a, b), f"utterance {u}: first mismatch at {np.argwhere(a != b)[:3]}"


@pytest.mark.parametrize("mode", MODES)
def test_unbatched_ragged_injected_noise(models, sds, mode):
    """six unbatched utterances of 7 .. 40 frames (a pair of equal length, a 1-frame-longer neighbour, several shorter than
    the longest's chunks): each row == the single call == the C twin, and a row that has ended writes nothing past its end"""
    model = models[mode]
    lengths = [7, 12, 12, 13, 27, 40]
    mels = _mels(lengths)
    noise = [_noise(mode, 200 * T, 1, 100 + u) for u, T in enumerate(lengths)]
    sentinel = -7
    many = model.generate_many_device(mels, False, 8000, 400, noise=noise, prefill=sentinel)
    _same(many, [_single(model, m, False, 8000, 400, n) for m, n in zip(mels, noise)])
    buf = many[0]._base
    assert buf.shape == (6, 8000)
    for u, T in enumerate(lengths):
        row = many[u]._base[many[u].storage_offset() // 8000]
        assert bool((row[200 * T:] == sentinel).all()) and bool((row[:200 * T] != sentinel).any())
    weights = {k: v.numpy() for k, v in sds[mode].items() if v.dtype == torch.float32}
    twin = mo.MolTwin(weights) if mode == "MOL" else wo.Twin(weights)
    aux, melup = twin.condition(mels[0][0].numpy())
    ref = twin.generate(aux, melup, [0], 1400, noise[0].numpy())
    assert np.array_equal(many[0].cpu().numpy(), ref)


def test_single_utterance_loop_refuses_many(models):
    """a workspace conditioned with two utterances is refused by the single-utterance loop, before any device work"""
    from mockingbird_b200 import _lib

    model, L = models["RAW"], _lib.lib()
    mel_cat = torch.cat([m.reshape(-1) for m in _mels([5, 9], seed=11)]).to(model._device)
    frames = (C.c_int32 * 2)(5, 9)
    stream = C.c_void_p(torch.cuda.current_stream(model._device).cuda_stream)
    ws = _lib.workspace(L.mb_wavernn_workspace_bytes_multi(model._handle, 2, frames, 1, 1800), model._device, model)
    _lib.check(L.mb_wavernn_condition_multi(model._handle, C.c_void_p(mel_cat.data_ptr()), frames, 2, C.c_void_p(ws.data_ptr()),
                                            ws.numel(), stream))
    out = torch.empty(1, 1000, dtype=torch.int16, device=model._device)
    rc = L.mb_wavernn_generate_rows(model._handle, (C.c_int32 * 1)(0), 1, 1000, 0, 100, None, 1, 0, 0, C.c_void_p(out.data_ptr()),
                                    C.c_void_p(ws.data_ptr()), ws.numel(), stream)
    assert rc != 0 and "call mb_wavernn_condition on this workspace first" in L.mb_last_error().decode()


@pytest.mark.parametrize("mode", MODES)
def test_device_rng_keyed_per_utterance(models, mode):
    """the built-in generator is keyed by (utterance seed, fold within the utterance): folded and of different seeds"""
    model = models[mode]
    mels = _mels([3, 9, 5, 9], seed=4)
    seeds = [99, 7, 7, 12345678901]
    model.rng = "device"
    try:
        many = model.generate_many_device(mels, True, 300, 40, seeds=seeds)
        singles = []
        for m, s in zip(mels, seeds):
            model.seed = s
            singles.append(_single(model, m, True, 300, 40))
    finally:
        model.rng, model.seed = "torch", 0
    assert [int(x.shape[0]) for x in many] == [2, 6, 3, 6]
    _same(many, singles)


@pytest.mark.parametrize("mode", MODES)
def test_torch_stream_per_utterance_seeds(models, mode):
    """rng='torch', seeds=[s_u]: utterance u as under torch.manual_seed(s_u); the global generator is not touched"""
    model = models[mode]
    mels = _mels([5, 2, 8, 5], seed=5)
    seeds = [11, 12, 11, 2 ** 40 + 1]
    torch.manual_seed(321)
    before = torch.get_rng_state()
    many = model.generate_many_device(mels, False, 8000, 400, seeds=seeds)
    assert torch.equal(torch.get_rng_state(), before)
    singles = []
    for m, s in zip(mels, seeds):
        torch.manual_seed(s)
        singles.append(_single(model, m, False, 8000, 400))
    _same(many, singles)
    many_b = model.generate_many_device(mels, True, 300, 40, seeds=seeds)
    singles = []
    for m, s in zip(mels, seeds):
        torch.manual_seed(s)
        singles.append(_single(model, m, True, 300, 40))
    _same(many_b, singles)


@pytest.mark.parametrize("mode", MODES)
def test_torch_stream_drop_in(models, mode):
    """seeds=None: the samples of the Python loop of single calls under the global generator, which ends in the same state"""
    model = models[mode]
    mels = _mels([4, 6, 1, 6, 3], seed=6)
    torch.manual_seed(77)
    singles = [_single(model, m, False, 8000, 400) for m in mels]
    tail = torch.rand(5)
    torch.manual_seed(77)
    many = model.generate_many_device(mels, False, 8000, 400)
    assert torch.equal(torch.rand(5), tail)
    _same(many, singles)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("target,overlap,lengths", [(300, 40, [1, 4, 6, 7, 8]), (100, 12, [40, 3]), (100, 12, [40, 5, 40])])
def test_folded_mix(models, mode, target, overlap, lengths):
    """folded utterances of 1 to 5 folds side by side; more than 64 rows (two row blocks) and more than 128 rows (several
    rows per CTA)"""
    model = models[mode]
    mels = _mels(lengths, seed=7)
    folds = [wo.fold_geometry(200 * T, target, overlap)[0] for T in lengths]
    if target == 300:
        assert sorted(folds) == [1, 3, 4, 4, 5]
    else:
        assert sum(folds) > (64 if len(lengths) == 2 else 128)
    steps = target + 2 * overlap
    noise = [_noise(mode, steps, B, 200 + u) for u, B in enumerate(folds)]
    many = model.generate_many_device(mels, True, target, overlap, noise=noise)
    _same(many, [_single(model, m, True, target, overlap, n) for m, n in zip(mels, noise)])


def test_row_block_empties(models):
    """70 unbatched rows, 66 of which end after 200 steps: the second row block stops running, the 4 longer rows go on alone"""
    model = models["RAW"]
    lengths = [1] * 30 + [2] + [1] * 36 + [2, 2, 3]
    mels = _mels(lengths, seed=8)
    seeds = list(range(1000, 1000 + len(lengths)))
    calls = []
    model.rng = "device"
    try:
        many = model.generate_many_device(mels, False, 8000, 400, seeds=seeds, prefill=-7,
                                          progress_callback=lambda i, n, b, r: calls.append((i, n, b)))
        assert [c[:3] for c in calls] == [(0, 600, 70), (100, 600, 70), (200, 600, 4), (300, 600, 4), (400, 600, 1), (500, 600, 1)]
        for u in (0, 30, 31, 67, 69):
            model.seed = seeds[u]
            _same([many[u]], [_single(model, mels[u], False, 8000, 400)])
    finally:
        model.rng, model.seed = "torch", 0
    buf = many[0]._base.cpu().numpy()
    live = np.sort(np.array([200 * T for T in lengths]))[::-1]
    for r in range(70):
        assert (buf[r, live[r]:] == -7).all() and (buf[r, :live[r]] >= 0).all()


def test_reference_golden_in_a_batch(models, golds):
    """the reference's fixture utterances, vocoded among other utterances under their own seed, reproduce the golden integer
    samples and the float64 waveform (RAW), both post-processing paths"""
    model, gold = models["RAW"], golds["RAW"]
    others = _mels([33, 26], seed=9)
    mels = [others[0], torch.from_numpy(gold["mel1"]), others[1]]
    idx = model.generate_many_device(mels, False, 8000, 400, seeds=[5, 1234, 6])
    assert np.array_equal(idx[1].cpu().numpy(), gold["idx1"])
    for post in ("device", "host"):
        model.post = post
        try:
            wavs = model.generate_many(mels, False, 8000, 400, True, seeds=[5, 1234, 6], progress_callback=lambda *a: None)
        finally:
            model.post = "device"
        assert model.training and wavs[1].dtype == np.float64 and wavs[1].shape == gold["wav1"].shape
        assert np.abs(wavs[1] - gold["wav1"]).max() <= 1e-12
        assert [len(w) for w in wavs] == [33 * 200, 27 * 200, 26 * 200]  # hop_length 256 never trims
    mels = [torch.from_numpy(gold["mel2"]), others[0]]
    wavs = model.generate_many(mels, True, 1000, 100, True, seeds=[1234, 8], progress_callback=lambda *a: None)
    assert np.abs(wavs[0] - gold["wav2"]).max() <= 1e-12
    with pytest.raises(ValueError, match="shorter than the 5120-sample fade-out"):
        model.generate_many(_mels([30, 25]), False, 8000, 400, True)


def test_reference_golden_in_a_batch_mol(models, golds):
    model, gold = models["MOL"], golds["MOL"]
    seed = json.loads(str(gold["meta"]))["gen_seed"]
    mels = [_mels([29], seed=10)[0], torch.from_numpy(gold["mel1"])]
    x = model.generate_many_device(mels, False, 1000, 100, seeds=[3, seed])
    assert np.abs(x[1].cpu().numpy() - gold["x1"]).max() <= TOL_MOL
    wavs = model.generate_many([torch.from_numpy(gold["mel2"]), mels[0]], True, 1000, 100, True, seeds=[seed, 3],
                               progress_callback=lambda *a: None)
    assert wavs[0].shape == gold["wav2"].shape and np.abs(wavs[0] - gold["wav2"]).max() <= TOL_MOL


def test_inference_module_protocol(sds, golds):
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    gold = golds["RAW"]
    rnn_vocoder._model = None
    with pytest.raises(Exception, match="Please load Wave-RNN"):
        rnn_vocoder.infer_waveforms([np.zeros((80, 30), np.float32)])
    rnn_vocoder.load_state(sds["RAW"])
    g = np.random.default_rng(0)
    mels = [gold["mel2"][0] * 4.0] + [g.uniform(-4, 4, (80, T)).astype(np.float32) for T in (26, 41, 30)]
    seeds = [1234, 1, 2, 3]
    quiet = lambda *a: None
    wavs = rnn_vocoder.infer_waveforms(mels, target=1000, overlap=100, seeds=seeds, progress_callback=quiet)
    assert [len(w) for w in wavs] == [6700, 5600, 8900, 6700]  # folds * 1100 + 100
    assert np.abs(wavs[0] - gold["wav2"]).max() <= 1e-12
    torch.manual_seed(2)
    one, sr = rnn_vocoder.infer_waveform(mels[2], target=1000, overlap=100, progress_callback=quiet)
    assert sr == 16000 and np.array_equal(one, wavs[2])
    split = rnn_vocoder.infer_waveforms(mels, target=1000, overlap=100, seeds=seeds, max_rows=11, progress_callback=quiet)
    assert all(np.array_equal(a, b) for a, b in zip(split, wavs))
    raw = rnn_vocoder.infer_waveforms([m / 4.0 for m in mels[:2]], normalize=False, target=1000, overlap=100, seeds=seeds[:2],
                                      progress_callback=quiet)
    assert all(np.array_equal(a, b) for a, b in zip(raw, wavs[:2]))
    rnn_vocoder._model = None
