"""Tacotron.generate_stream / Synthesizer.synthesize_spectrograms_stream on the GPU: every text's result is bitwise what
generate_many returns for it, whatever the slot count, the list order, the masks or the GST mode, with rows refilled mid-loop."""
import numpy as np
import pytest
import torch

import ref_init as ri

pytestmark = pytest.mark.gpu
R = 2


@pytest.fixture(scope="module")
def sd():
    return ri.tacotron_state_dict(0, r=R, randomize_bn=True)


@pytest.fixture(scope="module")
def model(sd):
    from mockingbird_b200.synthesizer.inference import Synthesizer

    return Synthesizer("unused.pt", verbose=False).load_state(sd)


def _texts(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    seqs = [torch.randint(2, 75, (n,), generator=g) for n in lengths]
    emb = torch.rand(len(lengths), 256, generator=g)
    return seqs, emb / emb.norm(dim=1, keepdim=True)


def _masks(lengths, caps, seed):
    g = torch.Generator().manual_seed(seed)
    enc = [torch.rand(2, n, 256, generator=g) < 0.5 for n in lengths]
    dec = [torch.rand(-(-c // R), 2, 256, generator=g) < 0.5 for c in caps]
    return enc, dec


def _equal(a, b):
    return all(x.shape == y.shape and torch.equal(x, y) for x, y in zip(a, b))


def _stream(model, *args, **kw):
    got = {}
    for i, mel, lin, attn in model.generate_stream(*args, **kw):
        assert i not in got, i  # every index exactly once
        got[i] = (mel, lin, attn)
    return got


def _list(n, seed, max_chars):
    """n texts with mixed caps: rows that end inside the first 16 steps, cap 1, a 1-character text and the longest accepted"""
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(2, 131, (n,), generator=g).tolist()
    caps = torch.randint(8, 81, (n,), generator=g).tolist()
    lengths[0], caps[0] = max_chars, 24
    lengths[1], caps[1] = 1, 30
    caps[2], caps[3], caps[4] = 1, 2, 20
    return lengths, caps


def test_bitwise_generate_many_mixed_caps_and_slots(model):
    m = model
    from mockingbird_b200 import _lib

    max_chars = int(_lib.lib().mb_tacotron_max_chars())
    lengths, caps = _list(130, 3, max_chars)
    seqs, emb = _texts(lengths, 4)
    seeds = [500 + 3 * i for i in range(len(seqs))]
    kw = dict(steps=caps, style_idx=-1, min_stop_token=4, seeds=seeds)
    ref = m.generate_many(seqs, emb, **kw)
    got = _stream(m, seqs, emb, **kw)
    assert sorted(got) == list(range(len(seqs)))
    early = 0
    for i in range(len(seqs)):
        assert _equal(got[i], ref[i]), i
        early += got[i][0].shape[1] < -(-caps[i] // R) * R
    assert early > 0  # the stop rule, not only the caps, ended rows
    sub = list(range(12))
    for slots in (1, 3, 8):
        got = _stream(m, [seqs[i] for i in sub], emb[sub], steps=[caps[i] for i in sub], style_idx=-1, min_stop_token=4,
                      seeds=[seeds[i] for i in sub], slots=slots)
        for i in sub:
            assert _equal(got[i], ref[i]), (slots, i)
    perm = list(range(40))[::-1]
    got = _stream(m, [seqs[i] for i in perm], emb[perm], steps=[caps[i] for i in perm], style_idx=-1, min_stop_token=4,
                  seeds=[seeds[i] for i in perm], slots=16)
    for k, i in enumerate(perm):
        assert _equal(got[k], ref[i]), ("perm", i)


@pytest.mark.parametrize("style_idx", [-1, 3])
def test_bitwise_with_injected_masks(model, style_idx):
    m = model
    lengths = [5, 130, 17, 64, 33, 101, 9, 48, 1, 77]
    caps = [40, 60, 24, 1, 50, 36, 60, 44, 20, 3]
    seqs, emb = _texts(lengths, 11)
    masks = _masks(lengths, caps, 12)
    kw = dict(steps=caps, style_idx=style_idx, min_stop_token=4, dropout_masks=masks)
    ref = m.generate_many(seqs, emb, **kw)
    for slots in (3, 128):
        got = _stream(m, seqs, emb, slots=slots, **kw)
        for i in range(len(seqs)):
            assert _equal(got[i], ref[i]), (slots, i)


def test_abandoned_stream_leaves_the_model_usable(model):
    m = model
    seqs, emb = _texts([40, 25, 70, 12, 90, 33], 31)
    caps = [30, 60, 30, 44, 60, 20]
    before = m.generate_many(seqs, emb, steps=caps, min_stop_token=4)
    it = m.generate_stream(seqs, emb, steps=caps, min_stop_token=4, slots=2)
    first = next(it)
    assert _equal(first[1:], before[first[0]])
    it.close()
    after = m.generate_many(seqs, emb, steps=caps, min_stop_token=4)
    for a, b in zip(before, after):
        assert _equal(a, b)


def test_synthesizer_surface_and_argument_errors(tmp_path, sd):
    from mockingbird_b200.synthesizer import inference

    path = tmp_path / "synth.pt"
    torch.save({"model_state": sd}, path)
    s = inference.Synthesizer(path, verbose=False)
    texts = ["ni hao", "zhe shi yi ge ce shi ju zi", "hello world and more words here", "a"]
    emb = [np.random.default_rng(i).random(256).astype(np.float32) for i in range(4)]
    specs = s.synthesize_spectrograms_many(texts, emb, steps=40, seeds=[9, 8, 7, 6])
    got = dict(s.synthesize_spectrograms_stream(texts, emb, steps=40, seeds=[9, 8, 7, 6], slots=2))
    assert sorted(got) == [0, 1, 2, 3]
    for i, spec in enumerate(specs):
        assert got[i].shape == spec.shape and np.array_equal(got[i], spec)
    m = s._model
    bad = [
        (([[]], torch.rand(1, 256)), {}),
        (([[5] * 5000], torch.rand(1, 256)), {}),
        (([[5, 6], [7]], torch.rand(2, 256)), {"seeds": [1]}),
        (([[5, 6], [7]], torch.rand(2, 256)), {"steps": [10, 10, 10]}),
        (([[5, 6], [7]], torch.rand(3, 256)), {}),
        (([[5, 6], [7]], torch.rand(2, 256)), {"steps": [10, 0]}),
    ]
    for args, kw in bad:
        with pytest.raises(ValueError) as many:
            m.generate_many(*args, **kw)
        with pytest.raises(ValueError) as stream:
            m.generate_stream(*args, **kw)  # raised before the first result is asked for
        assert str(many.value) == str(stream.value)
    for slots in (0, 129):
        with pytest.raises(ValueError):
            m.generate_stream([[5, 6]], torch.rand(1, 256), slots=slots)
    with pytest.raises(ValueError):
        s.synthesize_spectrograms_stream(texts, emb[:3])
