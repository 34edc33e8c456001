"""GPU tests of the per-row step origin of streamed decoding (row_start / ring), one launch at a time through mb_taco_debug and
mb_taco_tc_debug: a row that started at global step t0 reads and writes at its own step (global step - t0) modulo the ring, and
gives the same bits as the same row launched at that step without a start array.  Buffers are NaN-filled, so a write outside
the row's slot shows."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
RING = 7


def _dbg(kind, **k):
    from mockingbird_b200.synthesizer.taco_debug import parse_report, taco_debug

    return parse_report(taco_debug(kind, **k))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32, device="cuda")


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _f32(a):
    return np.asarray(a, np.float32)


def _same(a, b, name):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name


G = 40                           # the global step of the launches below
STARTS = [40, 39, 33, 30, 0, 25]  # own steps 0, 1, 7, 10, 40, 15: slots 0, 1, 0, 3, 5, 1 of a 7-step ring


def _own(b):
    return G - STARTS[b]


def test_lsa_step_and_ctx_at_the_rows_own_step():
    g = np.random.default_rng(1)
    B, Tc, D, S = len(STARTS), 45, 128, 512
    lens = [45, 3, 30, 1, 17, 45]
    inside = np.arange(Tc)[None, :] < np.array(lens)[:, None]
    chars = np.where(inside, g.integers(1, 75, (B, Tc)), 0).astype(np.int32)
    proj, seq = _f32(g.standard_normal((B, Tc, D)) * 0.5), _f32(g.standard_normal((B, Tc, S)))
    cum = np.where(inside, g.random((B, Tc)) * 2, 0).astype(np.float32)
    w = dict(conv_w=_f32(g.standard_normal((32, 1, 31)) * 0.3), conv_b=_f32(g.standard_normal(32) * 0.3),
             Lw=_f32(g.standard_normal((D, 32)) * 0.2), vw=_f32(g.standard_normal((1, D)) * 0.5), q=_f32(g.standard_normal((B, D))),
             Wq=_f32(g.standard_normal((D, D)) * 0.1), bq=_f32(g.standard_normal(D) * 0.1))
    d = {k: _cuda(v) for k, v in dict(w, proj=proj, seq=seq, chars=chars).items()}
    ld = RING * Tc
    sp = _i32([G - 1])
    starts, lens_d = _i32(STARTS), _i32(lens)

    def step(row_start, scores, cum_d, step_j=1):
        _dbg("lsa_step", ins=[None, d["proj"], d["seq"], d["chars"], d["conv_w"], d["conv_b"], d["Lw"], d["vw"], d["q"], d["Wq"],
                              d["bq"]], outs=[cum_d, scores, None], n=[B, Tc, S, ld, 512], step_ptr=sp, step_j=step_j,
             row_len=lens_d, row_start=row_start, ring=RING if row_start is not None else 0)

    scores, cum_d = _nan(B * ld), _cuda(cum)
    step(starts, scores, cum_d)
    sc = scores.cpu().numpy().reshape(B, RING, Tc)
    for b in range(B):
        ref_sc, ref_cum = _nan(B * ld), _cuda(cum)
        # the same row without a start array, at step own % RING (the padded path indexes the buffers by the step directly)
        step(None, ref_sc, ref_cum, step_j=_own(b) % RING - (G - 1))
        r = ref_sc.cpu().numpy().reshape(B, RING, Tc)
        slot = _own(b) % RING
        _same(sc[b, slot], r[b, slot], ("lsa_step scores", b))
        assert np.isnan(np.delete(sc[b], slot, axis=0)).all(), ("lsa_step wrote outside its slot", b)
        _same(cum_d.cpu().numpy()[b], ref_cum.cpu().numpy()[b], ("lsa_step cum", b))
    rows_pad, KB = 64, S // 64
    ctx = _nan(B, S)
    tiles = [torch.zeros(KB * rows_pad * 64, dtype=torch.int16, device="cuda") for _ in range(4)]
    _dbg("lsa_ctx", ins=[scores, d["seq"]], outs=[ctx] + tiles, n=[B, Tc, S, ld, rows_pad], step_ptr=sp, step_j=1, row_len=lens_d,
         row_start=starts, ring=RING)
    c = ctx.cpu().numpy()
    for b in range(B):
        slot = _own(b) % RING
        a = sc[b, slot, :lens[b]].astype(np.float64)
        ref = a @ seq[b, :lens[b]].astype(np.float64)
        assert np.abs(c[b] - ref).max() <= 1e-5 * (np.abs(a) @ np.abs(seq[b, :lens[b]])).max() + 1e-6, b
        one = _nan(1, S)
        sc1 = _cuda(sc[b:b + 1, slot].reshape(-1))
        _dbg("lsa_ctx", ins=[sc1, d["seq"][b:b + 1].contiguous()], outs=[one, None, None, None, None], n=[1, Tc, S, Tc, 64],
             row_len=lens_d[b:b + 1])
        _same(c[b], one.cpu().numpy()[0], ("lsa_ctx", b))


def test_prenet_reads_the_rows_own_frame_and_masks():
    g = np.random.default_rng(2)
    B, K, H, r = len(STARTS), 80, 256, 2
    x_ld = RING * r * K
    mel = _f32(g.standard_normal(B * x_ld + K))
    first = np.zeros(K, np.float32)
    W1, b1 = _f32(g.standard_normal((H, K)) * 0.1), _f32(g.standard_normal(H) * 0.1)
    W2, b2 = _f32(g.standard_normal((H, H)) * 0.1), _f32(g.standard_normal(H) * 0.1)
    m = (g.random((RING, 2, B, H)) < 0.5).astype(np.uint8)
    md, xd = _cuda(m), _cuda(mel)  # x + s * x_step is frame s * r - 1 of a ring that starts one frame into the buffer
    args = [None, _cuda(first), _cuda(W1), _cuda(b1), _cuda(W2), _cuda(b2), md, md[0, 1]]
    sp = _i32([G])
    y = _nan(B, H)
    _dbg("prenet", ins=[xd] + args[1:], outs=[y, None, None], n=[B, K, H, H, x_ld, r * K, 2 * B * H, 0, 64], step_ptr=sp,
         row_start=_i32(STARTS), ring=RING)
    got = y.cpu().numpy()
    for b in range(B):
        s = _own(b)
        ref = _nan(B, H)
        # without a start array: the row's frame and masks sit at index (s - 1) % RING + 1 and s % RING of the padded layout;
        # step 0 of the row reads the go frame
        if s == 0:
            _dbg("prenet", ins=[xd] + args[1:], outs=[ref, None, None], n=[B, K, H, H, x_ld, r * K, 2 * B * H, 0, 64])
        else:
            q = (s - 1) % RING + 1
            mq = np.zeros((RING + 1, 2, B, H), np.uint8)
            mq[q] = m[s % RING]  # the row's masks where the padded path looks at step q
            mq = _cuda(mq)
            _dbg("prenet", ins=[xd, args[1], args[2], args[3], args[4], args[5], mq, mq[0, 1]], outs=[ref, None, None],
                 n=[B, K, H, H, x_ld, r * K, 2 * B * H, 0, 64], step_ptr=_i32([q]))
        _same(got[b], ref.cpu().numpy()[b], ("prenet", b, s))


def test_stop_rule_at_the_rows_own_step():
    """the rule's t > 10 and cap apply to the row's own step; done steps are its own; no flags are written"""
    B, r, K = len(STARTS), 2, 64
    stopv = _cuda(np.full(B, 0.9, np.float32))  # every row passes the threshold
    caps = _i32([50, 50, 5, 50, 41, 16])
    for kern in ("stop_flag", "stop_step"):
        done = _i32([-1] * B)
        if kern == "stop_flag":
            _dbg("stop_flag", ins=[stopv], outs=[None], n=[B, r], fval=5.0, step_ptr=_i32([G]), row_done=done, row_caps=caps,
                 row_start=_i32(STARTS), ring=RING)
        else:
            x = _cuda(np.ones((B, K), np.float32))
            w = _cuda(np.full(K, 0.05, np.float32))
            y = _nan(B)
            _dbg("stop_step", segs=[dict(x=x, K=K, ld=K)], W=w, ldw=K, M=B, N=1, y=y, ldy=1,
                 outs=[None, torch.zeros(1, dtype=torch.int32, device="cuda")], n=[B, r], fval=5.0, step_ptr=_i32([G]),
                 row_done=done, row_caps=caps, row_start=_i32(STARTS), ring=RING)
        # own steps 0, 1, 7, 10, 40, 15: every row passes, so a row ends where its own t = 2 s > 10 (from step 6 on)
        want = [-1, -1, 7, 10, 40, 15]
        assert done.cpu().tolist() == want, (kern, done.cpu().tolist())


def test_skinny_plain_writes_the_rows_own_slab():
    from mockingbird_b200.synthesizer.tc_debug import tc_debug

    g = np.random.default_rng(3)
    M, N, K = len(STARTS), 160, 128
    A, W = _f32(g.standard_normal((M, K))), _f32(g.standard_normal((N, K)) * 0.05)
    Ad, Wd = _cuda(A), _cuda(W)
    slabs = _nan(RING, M, N)
    tc_debug("plain", M=M, N=N, K0=K, w=[Wd], x=[Ad], ldx=[K], y=slabs, ldy=N, step_ptr=_i32([G - 1]), step_j=1, y_step=M * N,
             row_start=_i32(STARTS), ring=RING)
    full = _nan(M, N)
    tc_debug("plain", M=M, N=N, K0=K, w=[Wd], x=[Ad], ldx=[K], y=full, ldy=N)
    out, ref = slabs.cpu().numpy(), full.cpu().numpy()
    for m in range(M):
        slot = _own(m) % RING
        _same(out[slot, m], ref[m], ("skinny", m))
        assert np.isnan(np.delete(out[:, m], slot, axis=0)).all(), m


def test_start_array_needs_a_ring():
    from mockingbird_b200 import _lib

    with pytest.raises(_lib.MbError):
        _dbg("stop_flag", ins=[_cuda(np.zeros(1, np.float32))], outs=[None], n=[1, 2], step_ptr=_i32([0]), row_done=_i32([-1]),
             row_caps=_i32([3]), row_start=_i32([0]), ring=0)


# ---- admission (admit_rows_kernel) on an open stream, through mb_tacotron_stream_regions ------------------------------------
_FILL = {0: 0xFF, 1: 0xFF, 2: 0xA5, 3: 0xA5}  # fp32 / fp16 planes NaN, int32 / uint8 a pattern no admission writes


def _tensor_at(ptr, n, dtype):
    """a device tensor aliasing n elements at ptr (through __cuda_array_interface__)"""
    class _A:
        __cuda_array_interface__ = {"shape": (n,), "typestr": {torch.float32: "<f4", torch.int16: "<i2", torch.uint8: "|u1",
                                                              torch.int32: "<i4"}[dtype], "data": (ptr, False), "version": 3}
    return torch.as_tensor(_A(), device="cuda")


def _regions(handle):
    import ctypes as C

    from mockingbird_b200 import _lib

    L = _lib.lib()
    n = L.mb_tacotron_stream_regions(handle, None, 0)
    arr = (_lib.TacoStreamRegion * n)()
    assert L.mb_tacotron_stream_regions(handle, arr, n) == n
    out = {}
    for g in arr:
        dt = {0: torch.float32, 1: torch.int16, 2: torch.uint8, 3: torch.int32}[g.kind]
        cnt = {0: g.rows * g.width, 1: -(-g.width // 64) * g.rows * 64, 2: g.depth * 2 * g.rows * g.width,
               3: g.rows * g.width}[g.kind]
        out[g.name.decode()] = (g, _tensor_at(g.ptr, cnt, dt))
    return out


def _tile_rows(t, g):
    """an fp16 operand plane as [rows, K] int16 (so.unpack_act_tiles: the chunk swizzle undone)"""
    import tc_split_oracle as so

    kb = -(-g.width // 64)
    return so.unpack_act_tiles(t.cpu().numpy().view(np.float16), g.rows, kb).view(np.int16)


def _rows(t, g):
    if g.kind == 1:
        return _tile_rows(t, g)
    if g.kind == 2:
        return t.cpu().numpy().reshape(g.depth, 2, g.rows, g.width)
    return t.cpu().numpy().reshape(g.rows, g.width)


def _fill(t, g):
    t.view(torch.uint8).fill_(_FILL[g.kind]) if t.dtype != torch.uint8 else t.fill_(_FILL[g.kind])


def _is_fill(a, kind):
    return np.all(np.ascontiguousarray(a).view(np.uint8) == _FILL[kind])


@pytest.fixture(scope="module")
def taco():
    import ref_init as ri

    from mockingbird_b200.synthesizer.inference import Synthesizer

    return Synthesizer("unused.pt", verbose=False).load_state(ri.tacotron_state_dict(0, r=2, randomize_bn=True))


def test_admission_resets_only_its_slot(taco):
    """admission into slot 1 of 3: every reset region's row of the slot becomes exactly the zeros a fresh row starts from, the
    slot's encoder rows, characters, length, cap, done step, start step and masks are written; every other row (other slots,
    the tile rows past the slots) keeps its NaN / pattern fill.  After the loop has run, a second admission into the same slot
    resets it again, and injected masks are copied for the row's own steps only."""
    import ctypes as C

    from mockingbird_b200 import _lib

    m = taco
    if not m._ready:
        m._upload()
    L = _lib.lib()
    S, Tc, max_steps, r = 3, 24, 40, 2
    need = int(L.mb_tacotron_stream_workspace_bytes(m._handle, S, Tc, max_steps, r))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    cur = torch.cuda.current_stream().cuda_stream
    h = C.c_void_p()
    _lib.check(L.mb_tacotron_stream_open(m._handle, S, Tc, max_steps, r, -1, C.c_float(10.0), C.c_void_p(ws.data_ptr()), need,
                                         C.c_void_p(cur), C.byref(h)))
    try:
        g = torch.Generator().manual_seed(7)
        lens = [24, 9, 1]
        chars = torch.zeros(3, Tc, dtype=torch.int32)
        for b, n in enumerate(lens):
            chars[b, :n] = torch.randint(2, 75, (n,), generator=g, dtype=torch.int32)
        chars = chars.cuda()
        spk = torch.rand(3, 256, generator=g).cuda()
        seeds = [11, 12, 13]
        _lib.check(L.mb_tacotron_stream_encode(h, 0, 3, C.c_void_p(chars.data_ptr()), C.c_void_p(spk.data_ptr()),
                                               (C.c_int32 * 3)(*lens), (C.c_uint64 * 3)(*seeds), None, C.c_void_p(cur)))
        torch.cuda.synchronize()
        regs = _regions(h)
        for name, (gr, t) in regs.items():
            if not name.startswith("pool"):
                _fill(t, gr)
        torch.cuda.synchronize()
        steps1 = 15  # 8 decoder steps

        def admit(slot, row, text, steps, masks=None):
            mp = None if masks is None else (C.c_void_p * 1)(masks.data_ptr())
            _lib.check(L.mb_tacotron_stream_admit(h, 1, (C.c_int32 * 1)(slot), (C.c_int32 * 1)(row), (C.c_int64 * 1)(text),
                                                  (C.c_int32 * 1)(lens[row]), (C.c_int32 * 1)(steps),
                                                  (C.c_uint64 * 1)(seeds[row]), mp, C.c_void_p(cur)))
            torch.cuda.synchronize()

        admit(1, 1, 5, steps1)
        cap = -(-steps1 // r)
        pool = {k: _rows(regs[k][1], regs[k][0]) for k in ("pool_seq", "pool_proj", "pool_chars")}
        for name, (gr, t) in regs.items():
            if name.startswith("pool"):
                continue
            a = _rows(t, gr)
            if gr.kind == 2:  # masks [ring][2][S][units]: the slot's first `cap` steps, drawn from its seed
                want = torch.zeros(2 * cap * gr.width, dtype=torch.uint8, device="cuda")
                rs = torch.tensor([seeds[1]], dtype=torch.int64, device="cuda")
                _dbg("fill_masks_seeded", outs=[want], n=[1, cap, gr.width, 1], row_seeds=rs)
                want = want.cpu().numpy().reshape(cap, 2, gr.width)
                assert np.array_equal(a[:cap, :, 1], want), name
                assert _is_fill(a[cap:, :, 1], 2) and _is_fill(np.delete(a, 1, axis=2), 2), name
                continue
            row, others = a[1], np.delete(a, 1, axis=0)
            assert _is_fill(others, gr.kind), (name, "a row outside the slot was written")
            if gr.reset:
                assert not row.any(), (name, "not reset to zero")
            elif name in ("seq", "proj", "chars"):
                _same_bytes = np.array_equal(np.ascontiguousarray(row).view(np.uint8),
                                             np.ascontiguousarray(pool["pool_" + name][1]).view(np.uint8))
                assert _same_bytes, (name, "not the staging-pool row")
            else:
                assert int(row[0]) == {"lens": lens[1], "caps": cap, "done": -1, "start": 0}[name], (name, int(row[0]))
        # give the free slots back what open gives them (one character, done at step 0) before the loop runs over every slot
        for name, val in (("lens", 1), ("caps", 1), ("done", 0), ("start", 0)):
            t = regs[name][1]
            t[0], t[2] = val, val
        regs["chars"][1].view(S, Tc)[[0, 2]] = 0
        # run the loop until the row stops, then refill the slot: its state is dirty now, and admission resets it again
        n_done, ids, frames, steps = C.c_int32(0), (C.c_int64 * S)(), (C.c_int32 * S)(), C.c_int64(0)
        _lib.check(L.mb_tacotron_stream_run(h, C.byref(n_done), ids, frames, C.byref(steps)))
        assert n_done.value == 1 and ids[0] == 5 and frames[0] == cap * r
        assert any(_rows(regs[k][1], regs[k][0])[1].any() for k in ("h1", "c1", "attn_h", "p3_hi.0", "p3_hi.1"))
        g2 = torch.Generator().manual_seed(8)
        inj = (torch.rand(cap + 3, 2, 256, generator=g2) < 0.5).to(torch.uint8).cuda()
        before = _rows(regs["dmask"][1], regs["dmask"][0]).copy()
        admit(1, 2, 6, steps1, masks=inj)
        for name, (gr, t) in regs.items():
            if gr.reset:
                assert not _rows(t, gr)[1].any(), (name, "refilled slot not reset")
        dm = _rows(regs["dmask"][1], regs["dmask"][0])
        assert np.array_equal(dm[:cap, :, 1], inj[:cap].cpu().numpy())  # only the row's own steps are copied
        assert np.array_equal(dm[cap:, :, 1], before[cap:, :, 1]) and np.array_equal(np.delete(dm, 1, 2), np.delete(before, 1, 2))
        assert int(_rows(regs["start"][1], regs["start"][0])[1, 0]) == steps.value
        assert int(_rows(regs["lens"][1], regs["lens"][0])[1, 0]) == lens[2]
    finally:
        L.mb_tacotron_stream_close(h)
