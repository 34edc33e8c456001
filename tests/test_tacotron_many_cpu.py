"""Why Tacotron.generate_many exists, shown on the CPU oracle, and its host-side batching plan."""
import pytest
import torch

import ref_init as ri
import tacotron_oracle as to
from mockingbird_b200.synthesizer.models.tacotron import MANY_CHUNK_ROWS, many_plan

TOL = 2e-4


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def test_padded_batch_rows_differ_from_the_utterance_alone():
    """In the reference's padded batch a short text's mel depends on its neighbours (padded characters take attention mass,
    the CBHG runs over the pad embedding, the backward GRU starts at the padded end): beyond the FP32 tolerance that
    generate_many is held to against the same utterance at B = 1 (2e-4)"""
    sd = ri.tacotron_state_dict(0, r=2, randomize_bn=True)
    g = torch.Generator().manual_seed(3)
    lengths, steps = [30, 12, 21], 20
    B, Tc, nst = len(lengths), max(lengths), steps // 2
    chars = torch.zeros(B, Tc, dtype=torch.long)
    for b, n in enumerate(lengths):
        chars[b, :n] = torch.randint(2, 75, (n,), generator=g)
    emb = torch.rand(B, 256, generator=g)
    emb = emb / emb.norm(dim=1, keepdim=True)
    enc = torch.rand(2, B, Tc, 256, generator=g) < 0.5
    dec = torch.rand(nst, 2, B, 256, generator=g) < 0.5
    masks = [enc[0], enc[1]] + [dec[s, j] for s in range(nst) for j in range(2)]
    mel_p, lin_p, _ = to.generate(sd, chars, emb, steps, 0, 10, masks, r=2)  # min_stop_token 10: every row runs `steps` frames
    for b in (1, 2):  # the padded rows
        n = lengths[b]
        mb = [enc[0][b:b + 1, :n], enc[1][b:b + 1, :n]] + [dec[s, j][b:b + 1] for s in range(nst) for j in range(2)]
        mel_1, lin_1, _ = to.generate(sd, chars[b:b + 1, :n], emb[b:b + 1], steps, 0, 10, mb, r=2)
        assert _rel(mel_p[b], mel_1[0]) > TOL, (b, _rel(mel_p[b], mel_1[0]))
        assert _rel(lin_p[b], lin_1[0]) > TOL, (b, _rel(lin_p[b], lin_1[0]))
    # the longest row has no padding: the batch changes it only by summation order
    mb = [enc[0][:1], enc[1][:1]] + [dec[s, j][:1] for s in range(nst) for j in range(2)]
    mel_1, _, _ = to.generate(sd, chars[:1], emb[:1], steps, 0, 10, mb, r=2)
    assert _rel(mel_p[0], mel_1[0]) <= TOL


def test_plan_sorts_longest_first_and_chunks():
    lengths = [5, 130, 17, 130, 64, 9]
    assert many_plan(lengths, 128) == [[1, 3, 4, 2, 5, 0]]
    assert many_plan(lengths, 4) == [[1, 3, 4, 2], [5, 0]]
    assert many_plan(lengths, 1) == [[1], [3], [4], [2], [5], [0]]
    assert many_plan([], 8) == []
    plan = many_plan(list(range(300)), MANY_CHUNK_ROWS)
    assert [len(c) for c in plan] == [128, 128, 44]
    assert sorted(i for c in plan for i in c) == list(range(300))
    for bad in (0, 129):
        with pytest.raises(ValueError):
            many_plan(lengths, bad)
