"""Tacotron.generate_many / Synthesizer.synthesize_spectrograms_many on the GPU: every utterance computed as its own B = 1
generate (oracle parity, one utterance at a time), bitwise the same whatever list, order or chunk it is run in, with dropout
keyed by the utterance's seed."""
import numpy as np
import pytest
import torch

import ref_init as ri
import tacotron_oracle as to

pytestmark = pytest.mark.gpu
TOL = 2e-4
R = 2


@pytest.fixture(scope="module")
def sd():
    return ri.tacotron_state_dict(0, r=R, randomize_bn=True)


@pytest.fixture(scope="module")
def model(sd):
    from mockingbird_b200.synthesizer.inference import Synthesizer

    return Synthesizer("unused.pt", verbose=False).load_state(sd)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


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


@pytest.mark.parametrize("style_idx", [-1, 3])
def test_vs_oracle_each_utterance_alone(sd, model, style_idx):
    """8 utterances of 5-130 characters with mixed caps and min_stop_token = 4 (the random-weight stop fires at different
    steps): each result matches the oracle run on that utterance alone, unpadded, with its own masks"""
    lengths = [5, 130, 17, 64, 33, 101, 9, 48]
    caps = [40, 60, 24, 60, 50, 36, 60, 44]
    seqs, emb = _texts(lengths, 11)
    enc, dec = _masks(lengths, caps, 12)
    outs = model.generate_many(seqs, emb, steps=caps, style_idx=style_idx, min_stop_token=4, dropout_masks=(enc, dec))
    stopped_early = 0
    for i, (mel, lin, attn) in enumerate(outs):
        nst = -(-caps[i] // R)
        masks = [enc[i][0][None], enc[i][1][None]] + [dec[i][s, j][None] for s in range(nst) for j in range(2)]
        mel_r, lin_r, attn_r = to.generate(sd, seqs[i][None].long(), emb[i][None], caps[i], style_idx, 4, masks, r=R)
        assert mel.shape == mel_r.shape[1:], (i, mel.shape, mel_r.shape)
        assert attn.shape == attn_r.shape[1:], (i, attn.shape, attn_r.shape)
        assert _rel(mel.cpu(), mel_r[0]) <= TOL, (i, _rel(mel.cpu(), mel_r[0]))
        assert _rel(lin.cpu(), lin_r[0]) <= TOL, (i, _rel(lin.cpu(), lin_r[0]))
        assert _rel(attn.cpu(), attn_r[0]) <= TOL, (i, _rel(attn.cpu(), attn_r[0]))
        stopped_early += mel.shape[1] < nst * R
    assert stopped_early > 0  # the per-row stop rule fired for some rows, not only the caps


def _equal(a, b):
    return all(x.shape == y.shape and torch.equal(x, y) for x, y in zip(a, b))


def _run(model, seqs, emb, caps, seeds, idx, masks=None):
    sub = None if masks is None else ([masks[0][i] for i in idx], [masks[1][i] for i in idx])
    return model.generate_many([seqs[i] for i in idx], emb[idx], steps=[caps[i] for i in idx], style_idx=-1,
                               min_stop_token=4, seeds=[seeds[i] for i in idx], dropout_masks=sub)


def test_bitwise_independent_of_list_order_and_chunks(model):
    """the same utterance gives the same bits in a 12-row list (1560 encoder rows), a permutation, subsets of 4 (240 rows)
    and 8 (800 rows), alone (< 64 rows), in a 70-row chunk and in a 130-utterance list (chunks of 128 and 2)"""
    lengths = [130, 20, 75, 5, 48, 110, 33, 60, 12, 90, 27, 100]
    caps = [60, 36, 20, 44, 60, 28, 52, 40, 24, 56, 32, 48]
    g = torch.Generator().manual_seed(5)
    fill_len = torch.randint(5, 131, (118,), generator=g).tolist()
    fill_caps = torch.randint(8, 61, (118,), generator=g).tolist()
    seqs, emb = _texts(lengths + fill_len, 21)
    caps = caps + fill_caps
    seeds = [1000 + 7 * i for i in range(len(seqs))]
    base = list(range(12))
    ref = _run(model, seqs, emb, caps, seeds, base)
    perm = [7, 2, 11, 0, 5, 9, 3, 1, 10, 6, 4, 8]
    runs = {
        "perm": perm,
        "sub4": [3, 8, 10, 7],       # 4 x 60 chars
        "sub8": [9, 4, 6, 1, 2, 7, 10, 11],
        "chunk70": list(range(70))[::-1],
        "all130": list(range(130)),
    }
    for name, idx in runs.items():
        out = _run(model, seqs, emb, caps, seeds, idx)
        got = {i: o for i, o in zip(idx, out)}
        for i in base:
            if i in got:
                assert _equal(got[i], ref[i]), (name, i)
    for i in (0, 3, 8):
        assert _equal(_run(model, seqs, emb, caps, seeds, [i])[0], ref[i]), ("single", i)
    # injected masks: the list, its permutation and single utterances
    masks = _masks(lengths, caps[:12], 22)
    ref_m = _run(model, seqs, emb, caps, seeds, base, masks)
    for i, o in zip(perm, _run(model, seqs, emb, caps, seeds, perm, masks)):
        assert _equal(o, ref_m[i]), ("masks perm", i)
    for i in (1, 5):
        assert _equal(_run(model, seqs, emb, caps, seeds, [i], masks)[0], ref_m[i]), ("masks single", i)


def test_seeds(model):
    seqs, emb = _texts([40, 25, 70], 31)
    caps = [30, 30, 30]
    a = model.generate_many(seqs, emb, steps=caps, seeds=[1, 2, 3], min_stop_token=10)
    b = model.generate_many(seqs, emb, steps=caps, seeds=[1, 2, 3], min_stop_token=10)
    c = model.generate_many(seqs, emb, steps=caps, seeds=[4, 5, 6], min_stop_token=10)
    for x, y, z in zip(a, b, c):
        assert _equal(x, y)
        assert not torch.equal(x[0], z[0])
    moved = model.generate_many([seqs[2], seqs[0]], emb[[2, 0]], steps=30, seeds=[3, 1], min_stop_token=10)
    assert _equal(moved[0], a[2]) and _equal(moved[1], a[0])
    default = model.generate_many(seqs, emb, steps=30, min_stop_token=10)
    assert _equal(default[1], model.generate_many([seqs[1]], emb[[1]], steps=30, seeds=[model.seed + 1], min_stop_token=10)[0])


def test_synthesizer_surface(tmp_path, sd):
    from mockingbird_b200.synthesizer import inference
    from mockingbird_b200.synthesizer.hparams import hparams
    from mockingbird_b200.synthesizer.utils.text import text_to_sequence

    path = tmp_path / "synth.pt"
    torch.save({"model_state": sd}, path)
    s = inference.Synthesizer(path, verbose=False)
    texts = ["ni hao", "zhe shi yi ge ce shi ju zi", "hello world and more words here", "a"]
    emb = [np.random.default_rng(i).random(256).astype(np.float32) for i in range(4)]
    specs, aligns = s.synthesize_spectrograms_many(texts, emb, return_alignments=True, steps=40, seeds=[9, 8, 7, 6])
    assert s.is_loaded() and len(specs) == len(aligns) == 4
    rev = s.synthesize_spectrograms_many(texts[::-1], emb[::-1], steps=40, seeds=[6, 7, 8, 9])[::-1]
    for a, b in zip(specs, rev):
        assert a.shape == b.shape and np.array_equal(a, b)
    t2 = texts
    if inference.lazy_pinyin is not None:
        t2 = [" ".join(inference.lazy_pinyin(v, style=inference.Style.TONE3, neutral_tone_with_five=True)) for v in texts]
    seqs = [text_to_sequence(t, hparams.tts_cleaner_names) for t in t2]
    raw = s._model.generate_many(seqs, torch.from_numpy(np.stack(emb)), steps=40, seeds=[9, 8, 7, 6])
    for spec, al, (_, lin, attn), q in zip(specs, aligns, raw, seqs):
        full = lin.cpu().numpy()
        n = spec.shape[1]
        assert np.array_equal(spec, full[:, :n])
        assert n == 0 or spec[:, -1].max() >= hparams.tts_stop_threshold
        assert (full[:, n:].max(axis=0) < hparams.tts_stop_threshold).all()
        assert al.shape == (full.shape[1] // R, len(q)) and np.array_equal(al, attn.cpu().numpy())
    m = s._model
    with pytest.raises(ValueError):
        m.generate_many([[]], torch.rand(1, 256))
    with pytest.raises(ValueError):
        m.generate_many([[5] * 5000], torch.rand(1, 256))
    with pytest.raises(ValueError):
        m.generate_many([[5, 6], [7]], torch.rand(2, 256), seeds=[1])
    with pytest.raises(ValueError):
        m.generate_many([[5, 6], [7]], torch.rand(2, 256), steps=[10, 10, 10])
    with pytest.raises(ValueError):
        m.generate_many([[5, 6], [7]], torch.rand(3, 256))
    with pytest.raises(ValueError):
        s.synthesize_spectrograms_many(texts, emb[:3])
