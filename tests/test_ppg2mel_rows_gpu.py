"""ppg2mel with one dropout stream per utterance (``inference_batch(seeds=)``, mb_ppg2mel_inference_rows): every row of a
many-utterance call is bitwise the utterance's own B = 1 ``inference(seed=s)`` call, whatever the call's size (one and two
library calls), order, sub-list or duplicates."""
import pytest
import torch

import ref_init as ri

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2

    m = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    m.load_state_dict(ri.ppg2mel_state_dict(0))
    m.eval()
    return m


@pytest.fixture(scope="module")
def pool():
    """130 utterances of 4-240 PPG frames, one speaker embedding each, and distinct 64-bit seeds"""
    g = torch.Generator().manual_seed(11)
    lengths = torch.randint(4, 241, (130,), generator=g).tolist()
    lengths[:3] = [4, 240, 7]
    utts = [(torch.randn(T, 144, generator=g).cuda(),
             torch.stack([torch.randn(T, generator=g), (torch.rand(T, generator=g) < 0.7).float()], 1).cuda())
            for T in lengths]
    spk = torch.randn(130, 256, generator=g).cuda()
    seeds = [int(s) for s in torch.randint(0, 1 << 62, (130,), generator=g)]
    seeds[5] = (1 << 64) - 1
    seeds[6] = 0
    return utts, spk, seeds


_alone = {}


def alone(model, pool, i, seed):
    """utterance i's B = 1 call with `seed` (cached)"""
    key = (i, seed)
    if key not in _alone:
        utts, spk, _ = pool
        ppg, lf0 = utts[i]
        mel, post, align = model.inference(ppg[None], lf0[None], spk[i:i + 1], seed=seed)
        _alone[key] = (mel.clone(), post.clone(), align.clone())
    return _alone[key]


def check(model, pool, idx, seeds):
    utts, spk, _ = pool
    outs = model.inference_batch([utts[i] for i in idx], spk[idx], seeds=seeds)
    assert len(outs) == len(idx)
    for r, (i, s) in enumerate(zip(idx, seeds)):
        mel, post, align = outs[r]
        ref = alone(model, pool, i, s)
        assert align.shape[0] == ref[2].shape[0], (r, i)  # decoder steps
        assert torch.equal(mel, ref[0]) and torch.equal(post, ref[1]) and torch.equal(align, ref[2]), (r, i)


@pytest.mark.parametrize("n", [1, 7, 128, 130])
def test_rows_equal_their_single_calls(model, pool, n):
    _, _, seeds = pool
    idx = list(range(n))
    check(model, pool, idx, [seeds[i] for i in idx])


def test_permutation_sublist_and_duplicates(model, pool):
    _, _, seeds = pool
    g = torch.Generator().manual_seed(3)
    perm = torch.randperm(130, generator=g).tolist()
    check(model, pool, perm, [seeds[i] for i in perm])
    sub = perm[17:40:3]
    check(model, pool, sub, [seeds[i] for i in sub])
    dup = [5, 5, 2, 9, 2, 5, 6]
    check(model, pool, dup, [seeds[i] for i in dup])
    # the same utterance twice with two seeds: each row follows its own seed
    check(model, pool, [1, 1, 0], [seeds[1], seeds[2], seeds[0]])


def test_seeds_change_the_draws(model, pool):
    """per-row seeds are live: one utterance with two seeds gives two different mels (the dropout is always on)"""
    utts, spk, _ = pool
    a = model.inference_batch([utts[1], utts[1]], spk[[1, 1]], seeds=[1, 2])
    assert a[0][0].shape != a[1][0].shape or not torch.equal(a[0][0], a[1][0])


def test_seed_path_keeps_row_keying(model, pool):
    """seed= still keys the draws by row (the stream of a row depends on its position): row 0 of a call is the B = 1 call
    with that seed, and the per-row mode with every seed equal reproduces it for row 0"""
    utts, spk, _ = pool
    idx = [3, 4, 8]
    old = model.inference_batch([utts[i] for i in idx], spk[idx], seed=77)
    new = model.inference_batch([utts[i] for i in idx], spk[idx], seeds=[77] * 3)
    order = sorted(range(3), key=lambda r: -utts[idx[r]][0].shape[0])
    first = order[0]  # the longest utterance is row 0 of the padded batch
    assert all(torch.equal(x, y) for x, y in zip(old[first], new[first]))
    assert all(torch.equal(x, y) for x, y in zip(new[first], alone(model, pool, idx[first], 77)))
