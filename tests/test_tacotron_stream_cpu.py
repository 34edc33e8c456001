"""The host scheduler of Tacotron.generate_stream: admission order, slot reuse, encoder batches and every text admitted once."""
import random

import pytest

from mockingbird_b200.synthesizer.models.tacotron import StreamSchedule, many_plan


def _drive(lengths, slots, seed):
    """run the schedule as generate_stream does, finishing random busy slots: -> (admissions, encodes) in event order"""
    rng = random.Random(seed)
    s = StreamSchedule(lengths, slots)
    admitted, encoded, busy = [], [], {}
    admitted_pos = 0
    while not s.done():
        for row0, batch in s.to_encode():
            # a batch goes to the half of the pool that the batch two before it used, after all of that batch was admitted
            k = len(encoded)
            assert row0 == (k % 2) * slots and batch == s.order[k * slots:(k + 1) * slots]
            assert admitted_pos >= (k - 1) * slots
            encoded.append(batch)
        for slot, text, row in s.admit():
            assert slot not in busy and 0 <= slot < slots
            k = admitted_pos // slots
            assert k < len(encoded) and row == (k % 2) * slots + admitted_pos % slots
            busy[slot] = text
            admitted.append((slot, text))
            admitted_pos += 1
        for slot in rng.sample(sorted(busy), rng.randint(1, len(busy))):
            s.finish(slot)
            del busy[slot]
    return s, admitted, encoded


@pytest.mark.parametrize("slots", [1, 3, 8, 128])
def test_admission_order_slot_reuse_and_encoding(slots):
    rng = random.Random(slots)
    lengths = [rng.randint(1, 150) for _ in range(300)]
    s, admitted, encoded = _drive(lengths, slots, slots)
    texts = [t for _, t in admitted]
    assert texts == [i for c in many_plan(lengths, 128) for i in c]  # longest first, ties in input order
    assert sorted(texts) == list(range(300))                          # every text admitted once
    assert [i for b in encoded for i in b] == texts                    # and encoded once, in that order
    used = {slot for slot, _ in admitted}
    assert used == set(range(min(slots, 300)))                         # slots are reused, none beyond `slots`


def test_lowest_free_slot_first_and_bad_slots():
    s = StreamSchedule([3, 9, 9, 1], 2)
    assert s.to_encode() == [(0, [1, 2]), (2, [0, 3])]  # both halves of the pool are free at the start
    assert s.admit() == [(0, 1, 0), (1, 2, 1)]
    s.finish(1)
    assert s.admit() == [(1, 0, 2)] and s.to_encode() == []
    s.finish(0)
    s.finish(1)
    assert s.admit() == [(0, 3, 3)]
    s.finish(0)
    assert s.done()
    for bad in (0, 129):
        with pytest.raises(ValueError):
            StreamSchedule([1], bad)
