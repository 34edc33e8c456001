"""Host logic of the multi-utterance WaveRNN loop (no GPU): the row table, where each utterance's noise starts in the
torch generator's stream, the multi-source MT19937 filler, the argument checks of the C ABI, utterance sharding on gloo."""
import ctypes as C
import multiprocessing as _mp
import os
import socket

import numpy as np
import pytest
import torch
import torch.nn as nn

from mockingbird_b200 import _lib
from mockingbird_b200.vocoder.wavernn.models.fatchord_version import CHUNK, RowPlan, WaveRNN, fold_geometry

ARGS = (512, 512, 9, 2, (5, 5, 8), 80, 128, 128, 10, 200, 16000)


def test_row_table_unbatched_ragged():
    """longest first, ties in input order; a 1-frame-longer neighbour; an utterance shorter than one chunk"""
    frames = [12, 40, 13, 12, 1, 27]
    p = RowPlan(frames, False, 8000, 400)
    assert p.order == [1, 5, 2, 0, 3, 4]
    assert p.frames == [40, 27, 13, 12, 12, 1]
    assert p.rows == 6 and p.max_steps == 8000
    assert p.row_steps.tolist() == [8000, 5400, 2600, 2400, 2400, 200]
    assert p.row_utt.tolist() == [0, 1, 2, 3, 4, 5] and p.row_fold.tolist() == [0] * 6 and p.row_start.tolist() == [0] * 6
    assert p.live(0) == (6, 6) and p.live(199) == (6, 6) and p.live(200) == (5, 5)
    assert p.live(2400) == (3, 3) and p.live(2599) == (3, 3) and p.live(2600) == (2, 2) and p.live(7999) == (1, 1)
    ch = p.chunks(CHUNK)
    assert len(ch) == 80 and ch[0] == (0, 100, 6, 6) and ch[1] == (100, 100, 6, 6) and ch[2] == (200, 100, 5, 5)
    assert ch[24] == (2400, 100, 3, 3) and ch[-1] == (7900, 100, 1, 1)
    # every row is alive in exactly the chunks that start before its end
    for r, s in enumerate(p.row_steps):
        assert sum(1 for c in ch if c[3] > r) == -(-int(s) // CHUNK)


def test_row_table_folded_mix():
    """batched: all rows have target + 2 * overlap steps, each utterance's folds are adjacent rows in input order"""
    frames = [9, 2, 7, 30]
    p = RowPlan(frames, True, 300, 40)
    folds = [fold_geometry(200 * T, 300, 40)[0] for T in frames]
    assert folds == [6, 2, 4, 18]
    assert p.order == [0, 1, 2, 3] and p.utt_rows == folds and p.utt_row0 == [0, 6, 8, 12] and p.rows == 30
    assert set(p.row_steps.tolist()) == {380} and p.max_steps == 380
    assert p.row_fold.tolist() == sum([list(range(b)) for b in folds], [])
    assert p.row_start.tolist() == sum([[340 * k for k in range(b)] for b in folds], [])
    assert p.row_utt.tolist() == sum([[u] * b for u, b in enumerate(folds)], [])
    assert p.chunks(CHUNK) == [(0, 100, 4, 30), (100, 100, 4, 30), (200, 100, 4, 30), (300, 80, 4, 30)]
    with pytest.raises(ValueError):
        RowPlan([5, 0], False, 8000, 400)


def test_workspace_grows_with_frames_and_row_blocks():
    h = WaveRNN(*ARGS)._handle
    L = _lib.lib()
    fr = lambda *a: (C.c_int32 * len(a))(*a)
    one = L.mb_wavernn_workspace_bytes_multi(h, 1, fr(30), 1, 6000)
    assert one == L.mb_wavernn_workspace_bytes(h, 30, 1, 6000) > 0
    for T, folds in ((2400, 58), (80, 65)):  # the single call is the one-utterance case
        assert L.mb_wavernn_workspace_bytes(h, T, folds, 8800) == L.mb_wavernn_workspace_bytes_multi(h, 1, fr(T), folds, 8800) > 0
    assert L.mb_wavernn_workspace_bytes_multi(h, 1, fr(30), 64, 6000) == one  # one row block
    assert L.mb_wavernn_workspace_bytes_multi(h, 1, fr(30), 65, 6000) > one
    assert L.mb_wavernn_workspace_bytes_multi(h, 2, fr(15, 15), 1, 3000) > one  # a second "past the end" row and padding
    assert L.mb_wavernn_workspace_bytes_multi(h, 2, fr(15, 0), 1, 3000) == 0
    assert L.mb_wavernn_workspace_bytes_multi(h, 1, fr(200000), 1, 100) == 0  # past the 32-bit indexing of the mel ladder
    assert L.mb_wavernn_workspace_bytes(h, 200000, 1, 100) == 0


def test_abi_argument_checks():
    """host-only refusals of the new entry points: status code and message, before any device work"""
    raw, mol = WaveRNN(*ARGS), WaveRNN(*ARGS, mode="MOL")
    L = _lib.lib()
    i32 = lambda *a: (C.c_int32 * len(a))(*a)
    u64 = lambda *a: (C.c_uint64 * len(a))(*a)
    p = C.c_void_p(256)  # never dereferenced: every call below is refused first

    def refused(status, text):
        assert status != 0
        assert text in L.mb_last_error().decode()

    refused(L.mb_wavernn_condition_multi(raw._handle, None, i32(5), 1, p, 1 << 30, None), "null argument")
    refused(L.mb_wavernn_condition_multi(raw._handle, p, i32(5, -1), 2, p, 1 << 30, None), "bad utterance lengths")
    refused(L.mb_wavernn_condition_multi(raw._handle, p, i32(5, 6), 2, p, 1024, None), "workspace too small")
    refused(L.mb_wavernn_condition_multi(raw._handle, p, i32(5, 6), 2, p, 1 << 30, None), "weights not finalized")
    refused(L.mb_wavernn_condition(raw._handle, None, 5, p, 1 << 30, None), "null argument")
    refused(L.mb_wavernn_condition(raw._handle, p, 200000, p, 1 << 30, None), "bad utterance lengths")

    def gen(fn, h, utt, start, steps, fold, max_steps, step0, n, n_live, noise=p, seeds=None):
        return fn(h, i32(*utt), i32(*start), i32(*steps), i32(*fold), len(utt), seeds, max_steps, step0, n, n_live, noise, p, p,
                  1 << 30, None)

    G, GM = L.mb_wavernn_generate_multi, L.mb_wavernn_generate_multi_mol
    refused(gen(GM, raw._handle, [0], [0], [200], [0], 200, 0, 100, 1), "not created in MOL mode")
    refused(gen(G, mol._handle, [0], [0], [200], [0], 200, 0, 100, 1), "MOL handle samples floats")
    refused(gen(G, raw._handle, [0], [0], [200], [0], 200, 0, 100, 1, noise=None), "null argument")  # neither noise nor seeds
    refused(gen(G, raw._handle, [0], [0], [200], [0], 200, 150, 100, 1), "step range")
    refused(gen(G, raw._handle, [0], [0], [200], [0], 200, 0, 129, 1), "step range")
    refused(gen(G, raw._handle, [0, -1], [0, 0], [200, 200], [0, 0], 200, 0, 100, 2), "outside the table")
    refused(gen(G, raw._handle, [0], [2 ** 31 - 100], [200], [0], 200, 0, 100, 1), "outside the table")  # start + step overflows
    refused(gen(G, raw._handle, [0, 1], [0, 0], [200, 400], [0, 0], 400, 0, 100, 2), "longest first")
    refused(gen(G, raw._handle, [0, 0], [0, 340], [380, 380], [0, 2], 380, 0, 100, 2), "folds of an utterance")
    refused(gen(G, raw._handle, [0, 1], [0, 0], [400, 200], [0, 0], 400, 200, 100, 2), "rows are alive")
    refused(gen(G, raw._handle, [0, 1], [0, 0], [400, 200], [0, 0], 400, 200, 100, 1, noise=None, seeds=u64(1, 2)),
            "weights not finalized")


def test_single_abi_argument_checks():
    """mb_wavernn_generate_rows[_mol] on an unfinalized handle: each bad argument is refused with its own message, before
    "weights not finalized" and before any launch"""
    raw, mol = WaveRNN(*ARGS), WaveRNN(*ARGS, mode="MOL")
    L = _lib.lib()
    i32 = lambda *a: (C.c_int32 * len(a))(*a)
    p = C.c_void_p(256)  # never dereferenced: every call below is refused first
    launches = L.mb_launch_count()

    def gen(m, starts, steps=200, step0=0, n=100, noise=p, noise_folds=None, row0=0):
        fn = L.mb_wavernn_generate_rows_mol if m.mode == "MOL" else L.mb_wavernn_generate_rows
        folds = len(starts) if noise_folds is None else noise_folds
        return fn(m._handle, i32(*starts), len(starts), steps, step0, n, noise, folds, row0, 0, p, p, 1 << 30, None)

    def refused(status, code, text):
        assert status == code, L.mb_last_error()
        assert text in L.mb_last_error().decode()

    for m in (raw, mol):
        refused(gen(m, [0, -1]), 1, "fold start -1 of row 1")
        refused(gen(m, [0, 2 ** 31 - 150]), 1, "fold start")
        refused(gen(m, [0, 340], noise_folds=3, row0=2), 1, "outside the 3 noise rows")
        refused(gen(m, [0], row0=-1, noise=None), 1, "outside the")
        refused(gen(m, [0], n=129), 1, "bad step range")
        refused(gen(m, [0], step0=150, n=100), 1, "bad step range")
        refused(gen(m, [0, 340], noise_folds=5, row0=3), 2, "weights not finalized")
    other = L.mb_wavernn_generate_rows_mol(raw._handle, i32(0), 1, 200, 0, 100, p, 1, 0, 0, p, p, 1 << 30, None)
    refused(other, 1, "not created in MOL mode")
    refused(L.mb_wavernn_generate_rows(mol._handle, i32(0), 1, 200, 0, 100, p, 1, 0, 0, p, p, 1 << 30, None), 1,
            "MOL handle samples floats")
    refused(L.mb_wavernn_generate(raw._handle, i32(-5), 1, 200, 0, 100, p, 0, p, p, 1 << 30, None), 1, "fold start -5")
    assert L.mb_launch_count() == launches


def _draw_reference(model, B, steps):
    """what WaveRNN.generate of the reference draws from the global generator for B rows x steps"""
    nn.GRUCell(512, 512)
    nn.GRUCell(512 + 32, 512)
    pos = torch.get_rng_state()
    for _ in range(steps):
        if model.mode == "RAW":
            torch.empty(B, 512).exponential_(1)
        else:
            torch.empty(1, B, 10).uniform_(1e-5, 1.0 - 1e-5)
            torch.empty(1, B).uniform_(1e-5, 1.0 - 1e-5)
    return pos


def _as_state(pos):
    """(state, left, next) -> the torch generator in that position"""
    from mockingbird_b200.vocoder.wavernn.models.fatchord_version import set_torch_cpu_generator_position

    set_torch_cpu_generator_position(*pos)
    return torch.get_rng_state()


@pytest.mark.parametrize("mode", ["RAW", "MOL"])
def test_noise_starts_drop_in(mode):
    """seeds=None: utterance u's noise starts where the sequence of single generate() calls starts it, and the generator
    ends where that sequence ends"""
    model = WaveRNN(*ARGS, mode=mode)
    blocks = [(1, 37), (3, 20), (2, 5), (1, 1)]
    torch.manual_seed(4321)
    want = [_draw_reference(model, B, steps) for B, steps in blocks]
    end = torch.get_rng_state()
    torch.manual_seed(4321)
    got = model.noise_starts(blocks, None)
    assert torch.equal(torch.get_rng_state(), end)
    for w, g in zip(want, got):
        assert torch.equal(_as_state(g), w)
    torch.set_rng_state(end)


@pytest.mark.parametrize("mode", ["RAW", "MOL"])
def test_noise_starts_seeded(mode):
    """seeds=[s_u]: manual_seed(s_u) + the two GRUCells; the global generator is left as it was"""
    model = WaveRNN(*ARGS, mode=mode)
    blocks, seeds = [(1, 50), (4, 9), (1, 50)], [7, 2 ** 35 + 3, 7]
    torch.manual_seed(99)
    before = torch.get_rng_state()
    got = model.noise_starts(blocks, seeds)
    assert torch.equal(torch.get_rng_state(), before)
    for s, g in zip(seeds, got):
        torch.manual_seed(s)
        nn.GRUCell(512, 512)
        nn.GRUCell(512 + 32, 512)
        want = torch.get_rng_state()
        assert torch.equal(_as_state(g), want)
    assert np.array_equal(got[0][0], got[2][0])
    with pytest.raises(ValueError):
        model.noise_starts(blocks, [1, 2])
    torch.set_rng_state(before)


def _position(seed, burn):
    from mockingbird_b200.vocoder.wavernn.models.fatchord_version import torch_cpu_generator_position

    torch.manual_seed(seed)
    torch.empty(burn).uniform_()
    return torch_cpu_generator_position()


@pytest.mark.parametrize("threads", [1, 3])
def test_fill_sources_equals_single_streams(threads):
    """three sources of different widths over two ragged chunks (the second source ends inside the first chunk, the third
    is gone in the second): every source's columns hold its own stream in order, untouched columns stay as they were"""
    L = _lib.lib()
    pos = [_position(s, b) for s, b in ((1, 0), (2, 100), (3, 623))]
    wps = np.array([1024, 2048, 22], np.uint64)
    col = np.array([0, 1024, 3072], np.uint64)
    total = [7 * 1024, 3 * 2048, 4 * 22]
    want = []
    for (state, left, nxt), n in zip(pos, total):
        st, l, x = state.copy(), C.c_int32(left), C.c_int32(nxt)
        out = np.empty(n, np.uint32)
        _lib.check(L.mb_mt19937_fill(st.ctypes.data, C.byref(l), C.byref(x), out.ctypes.data, n))
        want.append((out, st, l.value, x.value))
    states = np.stack([p[0] for p in pos]).astype(np.uint32)
    left = np.array([p[1] for p in pos], np.int32)
    nxt = np.array([p[2] for p in pos], np.int32)
    stride = 3094
    a = np.full((4, stride), 0xDEADBEEF, np.uint32)
    _lib.check(L.mb_mt19937_fill_sources(3, states.ctypes.data, left.ctypes.data, nxt.ctypes.data, wps.ctypes.data, col.ctypes.data,
                                         np.array([4, 3, 4], np.int32).ctypes.data, a.ctypes.data, stride, threads))
    b = np.full((3, 1024), 0xDEADBEEF, np.uint32)  # second chunk: only the first source is alive, the step is narrower
    _lib.check(L.mb_mt19937_fill_sources(1, states.ctypes.data, left.ctypes.data, nxt.ctypes.data, wps.ctypes.data, col.ctypes.data,
                                         np.array([3], np.int32).ctypes.data, b.ctypes.data, 1024, threads))
    assert np.array_equal(np.concatenate([a[:, :1024].ravel(), b.ravel()]), want[0][0])
    assert np.array_equal(a[:3, 1024:3072].ravel(), want[1][0]) and (a[3, 1024:3072] == 0xDEADBEEF).all()
    assert np.array_equal(a[:, 3072:].ravel(), want[2][0])
    for s in range(3):
        assert np.array_equal(states[s], want[s][1]) and (left[s], nxt[s]) == want[s][2:]
    assert L.mb_mt19937_fill_sources(1, states.ctypes.data, left.ctypes.data, nxt.ctypes.data, wps.ctypes.data, col.ctypes.data,
                                     np.array([1], np.int32).ctypes.data, b.ctypes.data, 1000, threads) != 0


def test_split_by_rows():
    from mockingbird_b200.vocoder.wavernn.inference import split_by_rows

    assert split_by_rows([6, 4, 8, 6], 9) == [[0], [1], [2], [3]]
    assert split_by_rows([6, 4, 8, 6], 10) == [[0, 1], [2], [3]]
    assert split_by_rows([6, 4, 8, 6], None) == [[0, 1, 2, 3]]
    assert split_by_rows([20, 1, 1], 4) == [[0], [1, 2]]
    assert split_by_rows([], 4) == []


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _FakeModel:
    """stands in for the device: the 'waveform' of an utterance depends on its mel and its seed only"""

    def generate_many(self, mels, batched, target, overlap, mu_law, seeds=None, progress_callback=None):
        return [np.full(int(m.shape[-1]) * 200, float(m.sum()) + s, np.float64) for m, s in zip(mels, seeds)]


def _shard_worker(rank, world, port, lengths, q):
    import torch.distributed as dist

    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    if world > 1:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rnn_vocoder._model = _FakeModel()
        mels = [np.full((80, T), 0.01 * (i + 1), np.float32) for i, T in enumerate(lengths)]
        seeds = [100 + i for i in range(len(lengths))]
        err = None
        if world > 1:
            try:
                rnn_vocoder.infer_waveforms(mels, batched=False)
            except ValueError as e:
                err = str(e)
        wavs = rnn_vocoder.infer_waveforms(mels, batched=False, seeds=seeds, max_rows=2)
        q.put((rank, err, None if wavs is None else [(len(w), float(w[0])) for w in wavs]))
    finally:
        if world > 1:
            dist.destroy_process_group()


def test_two_rank_utterance_sharding():
    """gloo world size 2: the utterances are dealt to the ranks, rank 0 returns them in input order, equal to the one-process
    result; without seeds the call is refused"""
    lengths = [30, 80, 22, 41, 64]
    ctx = _mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, lengths, q)) for r in range(2)]
    for p in procs:
        p.start()
    outs = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert outs[1][2] is None and all("per-utterance seeds" in o[1] for o in outs)
    q1 = ctx.Queue()
    p = ctx.Process(target=_shard_worker, args=(0, 1, 0, lengths, q1))
    p.start()
    single = q1.get(timeout=120)
    p.join(timeout=60)
    assert outs[0][2] == single[2]
    assert [n for n, _ in single[2]] == [200 * T for T in lengths]
