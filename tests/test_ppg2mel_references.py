"""float64 references of the ppg2mel decoder's kernels (oracle/ppg2mel_kernel_oracle.py) checked against ppg2mel_oracle's
torch fp32 arithmetic within their bounds, with wrong references (a k-tile dropped, the i / f gates swapped, the variance
over L - 1, the 1e-5 rule removed) falling outside them; whole models at feature widths the golden cases never reach; and
the MoL attention's shared-memory limit on T."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ppg2mel_kernel_oracle as ko
import ppg2mel_oracle as po
import ref_init as ri

gpu = pytest.mark.gpu


# ---- whole models at other feature widths ------------------------------------------------------------------------------------------
WIDTHS = [(1, 1), (37, 1024), (1024, 3)]


def _width_model(Dp, Ds):
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2

    sd = ri.ppg2mel_state_dict(0, bnf_dim=Dp, spk_dim=Ds)
    sd["decoder.stop_layer.linear_layer.weight"] = torch.zeros(1, 768)  # logit -1 every step: each row runs to 2 T_enc
    sd["decoder.stop_layer.linear_layer.bias"] = torch.full((1,), -1.0)
    m = MelDecoderMOLv2(**dict(ri.PPG2MEL_CONFIG, bottle_neck_feature_dim=Dp, spk_embed_dim=Ds)).cuda()
    m.load_state_dict(sd)
    return m.eval(), sd


def _width_utts(lengths, Dp, Ds, seed):
    gen = torch.Generator().manual_seed(seed)
    utts = [(torch.randn(T, Dp, generator=gen),
             torch.stack([torch.randn(T, generator=gen), (torch.rand(T, generator=gen) < 0.7).float()], 1)) for T in lengths]
    spk = torch.randn(len(lengths), Ds, generator=gen)
    masks = [(torch.rand(2 * (T // 4), 256, generator=gen) < 0.5, torch.rand(2 * (T // 4), 128, generator=gen) < 0.5)
             for T in lengths]
    return utts, spk, masks


@gpu
@pytest.mark.parametrize("Dp,Ds", WIDTHS)
def test_whole_model_feature_widths(Dp, Ds):
    m, sd = _width_model(Dp, Ds)
    utts, spk, masks = _width_utts([103, 57, 30], Dp, Ds, Dp + Ds)
    (ppg, lf0) = utts[0]
    one = m.inference(ppg[None], lf0[None], spk[:1], dropout_masks=masks[0])
    r = po.inference(sd, ppg, lf0, spk[0], masks=list(zip(*masks[0])))
    assert r["steps"] == one[2].shape[0]
    for name, got in (("mel", one[0]), ("mel_postnet", one[1]), ("alignments", one[2])):
        e = po.rel_errors(got.cpu(), r[name])
        print(f"model {Dp}/{Ds} {name}: {e}")
        assert e["max_rel"] <= 1e-3 and e["rms_rel"] <= 1e-3, (name, e)
    batch = m.inference_batch(utts, spk, dropout_masks=masks)
    for i, ((p, l), res) in enumerate(zip(utts, batch)):
        single = m.inference(p[None], l[None], spk[i:i + 1], dropout_masks=masks[i])
        assert all(torch.equal(a, b) for a, b in zip(res, single)), i


# ---- the attention's shared-memory limit -----------------------------------------------------------------------------------------
@gpu
def test_frames_over_the_attention_smem_limit_rejected():
    from mockingbird_b200 import _lib

    m, _ = _width_model(144, 256)
    utts, spk, masks = _width_utts([60], 144, 256, 9)
    before = m.inference(utts[0][0][None], utts[0][1][None], spk, dropout_masks=masks[0])
    L = _lib.lib()
    lo, hi = 4, 1 << 22  # frames accepted / refused by the workspace query
    assert L.mb_ppg2mel_workspace_bytes(m._handle, 1, lo) > 0 and L.mb_ppg2mel_workspace_bytes(m._handle, 1, hi) == 0
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if L.mb_ppg2mel_workspace_bytes(m._handle, 1, mid) else (lo, mid)
    te_max = lo // 4
    assert hi == 4 * (te_max + 1) and lo == 4 * te_max + 3
    optin = getattr(torch.cuda.get_device_properties(0), "shared_memory_per_block_optin", None)
    if optin is not None:  # the kernel's static arrays take well under 1 KB of it
        assert 4 * (2 * te_max + 1) <= optin < 4 * (2 * te_max + 3) + 1024, (te_max, optin)
    # the library call itself: refused before anything is queued, whatever buffers it was given
    small = torch.zeros(4096, device="cuda")
    ws = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    n0 = L.mb_launch_count()
    steps = (C.c_int32 * 1)()
    p = C.c_void_p(small.data_ptr())
    rc = L.mb_ppg2mel_inference(m._handle, p, p, p, (C.c_int32 * 1)(hi), 1, hi, None, None, C.c_uint64(0), p, p, p, p, steps,
                                C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == 1 and str(te_max).encode() in L.mb_last_error(), (rc, L.mb_last_error())
    assert L.mb_launch_count() == n0, "nothing may be launched"
    assert not small.any() and not ws.any()
    with pytest.raises(ValueError, match=str(te_max)):
        m.inference(torch.zeros(1, hi, 144), torch.zeros(1, hi, 2), spk)
    after = m.inference(utts[0][0][None], utts[0][1][None], spk, dropout_masks=masks[0])
    assert all(torch.equal(a, b) for a, b in zip(before, after)), "the handle stays usable"
    print(f"attention T_enc limit {te_max}")


# ---- CPU: the references against ppg2mel_oracle's torch fp32 arithmetic ------------------------------------------------------------
def _ok(got, ref, bound):
    return bool(np.all(np.abs(np.asarray(got, np.float64) - ref) <= bound))


@pytest.mark.parametrize("ks,s,p", [(1, 1, 0), (4, 2, 1), (5, 1, 2)])
def test_conv_reference_matches_torch(ks, s, p):
    g = np.random.default_rng(ks)
    B, T, Cin, N, lens = 3, 13, 6, 5, [13, 6, 1]
    x = g.standard_normal((B, T, Cin))
    w = g.standard_normal((N, Cin, ks))
    T_out = (T + 2 * p - ks) // s + 1
    lo = [(L + 2 * p - ks) // s + 1 if L + 2 * p >= ks else 0 for L in lens]
    ref, _ = ko.conv_gemm(x, lens, w.reshape(N, -1), ks, s, p, T_out, lo)
    for b, L in enumerate(lens):
        assert not ref[b, lo[b]:].any()
        if lo[b]:  # torch refuses an input shorter than the kernel
            t = F.conv1d(torch.from_numpy(x[b, :L].T[None]), torch.from_numpy(w), stride=s, padding=p)[0].T.numpy()
            assert np.allclose(ref[b, :lo[b]], t, rtol=1e-12, atol=1e-12)


def test_encoder_references_match_oracle():
    """each encoder stage of ppg2mel_oracle (torch fp32) against the reference on the same fp32 input, within the bound"""
    sd = ri.ppg2mel_state_dict(0)
    gen = torch.Generator().manual_seed(1)
    T = 37
    ppg, spk = torch.randn(T, 144, generator=gen), torch.randn(256, generator=gen)
    x = ppg.t()[None]
    h = F.leaky_relu(F.conv1d(x, sd["bnf_prenet.0.weight"]), 0.1)
    r, b = ko.conv_gemm(ppg.numpy()[None], [T], sd["bnf_prenet.0.weight"].numpy()[:, :, 0], 1, 1, 0, T, [T], act=1)
    assert _ok(h[0].T.numpy(), r[0], b[0])
    n = F.instance_norm(h, eps=1e-5)
    hx = h[0].T.numpy().astype(np.float64)
    r, b = ko.instance_norm(hx[None], [T])
    # torch takes the statistics in fp32 where the kernel uses double: charge its mean and variance sums too
    inv = 1 / np.sqrt(hx.var(0) + 1e-5)
    torch_stats = ko.gamma(2 * T) * (np.abs(hx).mean(0) + np.abs(hx - hx.mean(0))) * inv + ko.gamma(2 * T) * np.abs(r[0])
    assert _ok(n[0].T.numpy(), r[0], b[0] + torch_stats)
    assert not _ok(n[0].T.numpy(), r[0] * ((T - 1) / T) ** 0.5, b[0] + torch_stats), "variance over L - 1"
    c = F.leaky_relu(F.conv1d(n, sd["bnf_prenet.3.weight"], sd["bnf_prenet.3.bias"], 2, 1), 0.1)
    wk = sd["bnf_prenet.3.weight"].numpy()
    r, b = ko.conv_gemm(n[0].T.numpy()[None], [T], wk.reshape(256, -1), 4, 2, 1, T // 2, [T // 2],
                        bias=sd["bnf_prenet.3.bias"].numpy(), act=1)
    assert _ok(c[0].T.numpy(), r[0], b[0])
    # a reference that drops the last k-tile falls outside the bound
    r2, _ = ko.conv_gemm(n[0].T.numpy()[None], [T], wk.reshape(256, -1), 4, 2, 1, T // 2, [T // 2],
                         bias=sd["bnf_prenet.3.bias"].numpy(), act=1, drop_k=16)
    assert not _ok(c[0].T.numpy(), r2[0], b[0])
    # reduce_proj with the normalised speaker half as a per-row bias
    mem_in = torch.randn(9, 256, generator=gen)
    full = F.linear(torch.cat([mem_in, F.normalize(spk[None]).expand(9, -1)], -1), sd["reduce_proj.weight"],
                    sd["reduce_proj.bias"])
    rb, bb = ko.spk_bias(spk.numpy()[None], sd["reduce_proj.weight"].numpy(), sd["reduce_proj.bias"].numpy())
    r, b = ko.conv_gemm(mem_in.numpy()[None], [9], sd["reduce_proj.weight"].numpy()[:, :256], 1, 1, 0, 9, [9], bias=rb)
    assert _ok(full.numpy(), r[0], b[0] + bb)


def test_postnet_references_match_oracle():
    sd = ri.ppg2mel_state_dict(0)
    gen = torch.Generator().manual_seed(2)
    T = 21
    mel = torch.randn(T, 80, generator=gen)
    x = mel.t()[None]
    for i in range(5):
        pfx = f"postnet.convolutions.{i}"
        y = F.conv1d(x, sd[pfx + ".0.conv.weight"], sd[pfx + ".0.conv.bias"], 1, 2)
        y = F.batch_norm(y, sd[pfx + ".1.running_mean"], sd[pfx + ".1.running_var"], sd[pfx + ".1.weight"],
                         sd[pfx + ".1.bias"], False, 0.1, 1e-5)
        if i < 4:
            y = torch.tanh(y)
        w = sd[pfx + ".0.conv.weight"].numpy()
        bn = [sd[pfx + k].numpy() for k in (".1.running_mean", ".1.running_var", ".1.weight", ".1.bias")]
        r, b = ko.conv_gemm(x[0].T.numpy()[None], [T], w.reshape(w.shape[0], -1), 5, 1, 2, T, [T],
                            bias=sd[pfx + ".0.conv.bias"].numpy(), bn=bn, act=2 if i < 4 else 0,
                            res=mel.numpy()[None] if i == 4 else None)
        got = (y[0].T + mel).numpy() if i == 4 else y[0].T.numpy()
        assert _ok(got, r[0], b[0]), i
        x = y
    full = po.postnet(sd, mel)
    assert _ok(full.numpy(), r[0], b[0])


def test_decoder_step_references_match_oracle():
    """one decoder step of ppg2mel_oracle.inference (torch fp32) stage by stage against the references on the same inputs"""
    sd = ri.ppg2mel_state_dict(0)
    gen = torch.Generator().manual_seed(3)
    Te = 23
    memory = torch.randn(Te, 256, generator=gen)
    frame = torch.randn(1, 80, generator=gen)
    ah, ac = torch.tanh(torch.randn(1, 512, generator=gen)), torch.randn(1, 512, generator=gen)
    dh, dc = torch.tanh(torch.randn(1, 512, generator=gen)), torch.randn(1, 512, generator=gen)
    ctx = torch.randn(1, 256, generator=gen)
    mu = torch.rand(1, 5, generator=gen) * 3
    k1, k2 = torch.rand(256, generator=gen) < 0.5, torch.rand(128, generator=gen) < 0.5
    W1, W2 = sd["decoder.prenet.layers.0.linear_layer.weight"], sd["decoder.prenet.layers.1.linear_layer.weight"]
    x = F.relu(F.linear(frame, W1)) * (k1.float() * 2.0)
    x = F.relu(F.linear(x, W2)) * (k2.float() * 2.0)
    r, b = ko.prenet(frame.numpy(), W1.numpy(), W2.numpy(), k1.numpy()[None], k2.numpy()[None])
    assert _ok(x.numpy(), r, b)

    def lstm_ref(p, xin, ctx_, h, c, **kw):
        return ko.lstm(xin.numpy(), ctx_.numpy(), h.numpy(), c.numpy(), sd[p + ".weight_ih"].numpy(),
                       sd[p + ".weight_hh"].numpy(), (sd[p + ".bias_ih"].double() + sd[p + ".bias_hh"].double()).numpy(),
                       **kw)

    ah2, ac2 = po._lstm(torch.cat((x, ctx), -1), ah, ac, sd, "decoder.attention_rnn")
    (hr, cr), (eh, ec) = lstm_ref("decoder.attention_rnn", x, ctx, ah, ac)
    assert _ok(ah2.numpy(), hr, eh) and _ok(ac2.numpy(), cr, ec)
    (hr2, cr2), _ = lstm_ref("decoder.attention_rnn", x, ctx, ah, ac, swap_if=True)
    assert not (_ok(ah2.numpy(), hr2, eh) and _ok(ac2.numpy(), cr2, ec)), "swapped gates must fall outside the bound"
    qn = "decoder.attention_layer.query_layer"
    hq = F.relu(F.linear(ah2, sd[qn + ".0.weight"], sd[qn + ".0.bias"]))
    r, b = ko.query(ah2.numpy(), sd[qn + ".0.weight"].numpy(), sd[qn + ".0.bias"].numpy())
    assert _ok(hq.numpy(), r, b)
    params = F.linear(hq, sd[qn + ".2.weight"], sd[qn + ".2.bias"])
    alpha, mu2 = po.mol_alpha(params, mu, Te)
    a, da, mr, dmu = ko.mol_alpha(hq.numpy(), sd[qn + ".2.weight"].numpy(), sd[qn + ".2.bias"].numpy(), mu.numpy(), Te)
    assert _ok(mu2.numpy(), mr, dmu)
    assert ko.alpha_ok(alpha.numpy()[0], a[0], da[0]).all()
    c2 = torch.bmm(alpha.unsqueeze(1), memory.unsqueeze(0)).squeeze(1)
    r, b = ko.mol_context(a[0], da[0], memory.numpy(), got_alpha=alpha.numpy()[0])
    assert _ok(c2.numpy()[0], r, b)
    r, b = ko.mol_context(a[0], da[0], memory.numpy())
    assert _ok(c2.numpy()[0], r, b)
    dh2, dc2 = po._lstm(torch.cat((ah2, c2), -1), dh, dc, sd, "decoder.decoder_rnn_layers.0")
    (hr, cr), (eh, ec) = lstm_ref("decoder.decoder_rnn_layers.0", ah2, c2, dh, dc)
    assert _ok(dh2.numpy(), hr, eh) and _ok(dc2.numpy(), cr, ec)
    out = torch.cat((dh2, c2), 1)
    mel = F.linear(out, sd["decoder.linear_projection.linear_layer.weight"], sd["decoder.linear_projection.linear_layer.bias"])
    stop = F.linear(out, sd["decoder.stop_layer.linear_layer.weight"], sd["decoder.stop_layer.linear_layer.bias"])
    (mr, me), (sr, se) = ko.proj(dh2.numpy(), c2.numpy(), sd["decoder.linear_projection.linear_layer.weight"].numpy(),
                                 sd["decoder.linear_projection.linear_layer.bias"].numpy(),
                                 sd["decoder.stop_layer.linear_layer.weight"].numpy()[0],
                                 float(sd["decoder.stop_layer.linear_layer.bias"][0]))
    assert _ok(mel.numpy(), mr, me) and _ok(stop.numpy()[:, 0], sr, se)


def test_alpha_rule_reference_rejects_missing_rule():
    """wide-apart narrow mixtures: most fp32 alphas are exactly 0 and become 1e-5.  The oracle's alphas pass; the same
    alphas with the rule removed (0 kept) or with 2e-5 substituted do not"""
    Te = 60
    params = torch.tensor([[0.0, 1.0, -1.0, 0.5, 2.0] + [-4.0] * 5 + [3.0, 5.0, 8.0, 12.0, 20.0]])
    mu = torch.zeros(1, 5)
    alpha, _ = po.mol_alpha(params, mu, Te)
    a, da, _, _ = ko.mol_alpha(params.numpy(), np.eye(15), np.zeros(15), mu.numpy(), Te)  # W2 = I: the params themselves
    got = alpha.numpy()[0]
    sub = got == ko.EPS_MOL
    assert sub.sum() > Te // 2
    assert ko.alpha_ok(got, a[0], da[0]).all()
    assert not ko.alpha_ok(np.where(sub, 0.0, got), a[0], da[0]).all()
    assert not ko.alpha_ok(np.where(sub, np.float32(2e-5), got), a[0], da[0]).all()


def test_stop_decision_edges():
    assert ko.stop_decision(0.75, 1e-7, 9, 8) is False   # ns = mn - 1
    assert ko.stop_decision(0.75, 1e-7, 10, 8) is True   # ns = mn
    assert ko.stop_decision(-0.75, 1e-7, 9, 5) is True   # ns = mx
    assert ko.stop_decision(0.0, ko.TINY, 10, 8) is False  # an exact 0: sigmoidf(0) = 0.5 is not > 0.5
    assert ko.stop_decision(1e-9, 1e-7, 10, 8) is None
    assert ko.stop_decision(-0.75, 1e-7, 10, 8) is False
