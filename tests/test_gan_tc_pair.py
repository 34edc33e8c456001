"""GPU tests of the fused resblock pair (tc_conv_kernel<..., PAIR = true>) and of the tap conv's epilogue variants, launch by
launch (mb_gan_debug_launch), against the float64 references of oracle/tc_pair_oracle.py rounded where the kernel rounds.

Covered: every fusable (C, k, d) pair of HiFi-GAN and Fre-GAN (Fre-GAN's 16-channel stage carried with 32 channels) at lengths
around the work-item boundaries, ragged batches, persistent loops with more work items than SMs, EPI_STORE / EPI_ADD /
EPI_ADD_DIV with and without red.global.add, fp32 / activated fp16 / hi-lo residuals, plain and hi-lo fp16 output planes, the
pair fused vs as two launches, and every compiled kernel instance.
"""
import pytest
import torch

import ref_init as ri
import tc_pair_oracle as po

pytestmark = pytest.mark.gpu

SLOPE = 0.1
RAN = set()            # kernel instances (N, MT, CW, PAIR) launched by the tests of this module
WORST = {}             # pair signature -> worst |y - ref| / bound
BITWISE = {}           # pair signature -> fused == two launches bit for bit


def _make(kind, cfg, precision="f16tc"):
    from mockingbird_b200.vocoder.fregan.models import FreGAN
    from mockingbird_b200.vocoder.hifigan.models import Generator

    if kind == "fregan":
        sd = ri.rescale_variance_preserving(ri.fregan_state_dict(cfg, 0), 1.0)
        g = FreGAN(cfg, precision=precision)
    else:
        sd = ri.rescale_variance_preserving(ri.hifigan_state_dict(cfg, 0), 1.0)
        g = Generator(cfg, precision=precision)
    g.cuda()
    g.load_state_dict(sd)
    g.eval()
    g.remove_weight_norm()
    return g, sd


# a HiFi-GAN with k = 5 resblocks: its C = 128 layers plan MT = 1 (the only configuration that reaches <128, 1, 64>)
K5_CONFIG = dict(ri.HIFIGAN_CONFIG_16K, upsample_rates=[5, 5], upsample_kernel_sizes=[10, 10], upsample_initial_channel=256,
                 resblock_kernel_sizes=[5], resblock_dilation_sizes=[[1, 3, 5]])


@pytest.fixture(scope="module")
def gens():
    return {"hifigan": _make("hifigan", ri.HIFIGAN_CONFIG_16K), "fregan": _make("fregan", ri.FREGAN_CONFIG),
            "k5": _make("hifigan", K5_CONFIG)}


def _info(g, i):
    s = g.layer_info(i)
    return s.split()[1], {k: int(v) for k, v in (t.split("=") for t in s.split()[2:])}


def _weights(sd, name, cin, cout, transposed=False):
    """the checkpoint tensors zero-padded to the plan's channel counts (Fre-GAN's 16-channel stage runs with 32)"""
    w, b = sd[name + ".weight"].double(), sd[name + ".bias"].double()
    if transposed:
        wp = torch.zeros(cin, cout, w.shape[2], dtype=torch.float64)
    else:
        wp = torch.zeros(cout, cin, w.shape[2], dtype=torch.float64)
    wp[: w.shape[0], : w.shape[1]] = w
    bp = torch.zeros(cout, dtype=torch.float64)
    bp[: b.shape[0]] = b
    return wp.cuda(), bp.cuda()


def _pairs(g):
    """first fused pair (op index) of every distinct (C, k, dilation, padded) signature"""
    out, seen = [], set()
    for i in range(g.num_layers()):
        if g.layer_info(i).startswith("add"):
            continue
        p = g.tc_plan_info(i)
        if not p["fuse_next"]:
            continue
        name, d = _info(g, i)
        key = (d["cout"], d["k"], d["dil"])
        if key not in seen:
            seen.add(key)
            out.append((i, key, p))
    return out


def _pair_cases(gens):
    cases = []
    for kind in ("hifigan", "fregan"):
        g, _ = gens[kind]
        stages = {}
        for i, key, p in _pairs(g):
            cases.append((kind, i, key, p))
        # Fre-GAN: the 16-channel stage (carried with 32 channels) has its own pairs of the same (C, k, d)
        if kind == "fregan":
            for i in range(g.num_layers()):
                name, d = _info(g, i) if not g.layer_info(i).startswith("add") else (None, None)
                if name and ".convs1." in name and g.tc_plan_info(i)["fuse_next"] and d["rate_in"] == 200 and \
                        (d["k"], d["dil"]) not in stages:
                    stages[(d["k"], d["dil"])] = i
            cases += [(kind, i, (32, k, dd), g.tc_plan_info(i)) for (k, dd), i in sorted(stages.items())]
    return cases


def _run_pair(gens, kind, i, x, *, pair=1, res=None, res_kind="f32", mode="store", red_add=False, S=None, out16=None,
              lengths=None):
    g, sd = gens[kind]
    y, hi, lo, launches = g.debug_launch(i, x, pair=pair, mode=mode, div=3.0, red_add=red_add, y_init=S, residual=res,
                                         res_kind=res_kind if res is not None else None, res_slope=SLOPE, out16=out16,
                                         out_slope=SLOPE, lengths=lengths)
    for ln in launches:
        RAN.add(ln["kernel"])
    return y, hi, lo, launches


def _pair_ref(gens, kind, i, x, *, res=None, res_kind="f32", mode="store", S=None, valid=None):
    g, sd = gens[kind]
    n1, d1 = _info(g, i)
    n2, d2 = _info(g, i + 1)
    C = d1["cout"]
    w1, b1 = _weights(sd, n1, C, C)
    w2, b2 = _weights(sd, n2, C, C)
    y, mid, gap = po.pair_reference(x.double(), w1, b1, w2, b2, d1["dil"], SLOPE, SLOPE, res=res, res_kind=res_kind,
                                    res_slope=SLOPE, mode=mode, S=S, div=3.0, valid=valid)
    return y, po.pair_bound(y, w2, gap, mode, 3.0, valid)


def _check(y, ref, bound, what, key=None):
    r = po.worst_ratio(y, ref, bound)
    if key is not None:
        WORST[key] = max(WORST.get(key, 0.0), r)
    assert r <= 1.0, (what, r)


def _check_planes(y, hi, lo, valid, what):
    """hi == fp16(lrelu(y)) to one fp16 ulp, hi + lo == lrelu(y) to 2e-5 of the scale, everything past a length exactly 0"""
    a = po.act32(y, SLOPE)
    ulp = (po.q16(a.abs() * (1 + 2.0 ** -10)) - po.q16(a.abs())).abs().clamp_min(2.0 ** -24)
    assert bool(((hi.double() - po.q16(a)).abs() <= ulp).all()), what
    if lo is not None:
        assert float((hi.double() + lo.double() - a).abs().max()) <= po.TOL * float(a.abs().max()) + 1e-30, what
    if valid is not None:
        B, _, L = y.shape
        past = po.row_mask(B, L, valid, y.device) == 0
        for t in (y, hi, lo):
            if t is not None:
                assert bool((t.masked_select(past.expand_as(t)) == 0).all()), what


# ---------------------------------------------------------------------------------------------------------------------------------
def test_pairs_at_item_boundaries(gens):
    """every fusable pair signature: L in {1, h2, rows_item - 1, rows_item, rows_item + 1, 2 rows_item + h2}, then a ragged batch"""
    gen = torch.Generator().manual_seed(11)
    failures = []
    for kind, i, key, p in _pair_cases(gens):
        C, k, dil = key
        h2, ri_ = (k - 1) // 2, p["pair_rows_item"]
        sig = (kind, i) + key
        for L in sorted({1, h2, ri_ - 1, ri_, ri_ + 1, 2 * ri_ + h2}):
            x = torch.randn(1, C, L, generator=gen).cuda()
            res = torch.randn(1, C, L, generator=gen).cuda()
            y, _, _, ln = _run_pair(gens, kind, i, x, res=res)
            assert ln[0]["kernel"] == p["kernel"] and ln[0]["rows_item"] == ri_, (sig, ln)
            ref, bound = _pair_ref(gens, kind, i, x, res=res)
            r = po.worst_ratio(y, ref, bound)
            WORST[sig] = max(WORST.get(sig, 0.0), r)
            if not r <= 1.0:
                failures.append((sig, L, r))
        # ragged: lengths at an item boundary +- 1, 1, < h2 (rows past a length are zero in the input, as the producer leaves them)
        valid = [ri_ - 1, ri_ + 1, 1, h2 - 1]
        L = 2 * ri_ + h2
        x = torch.randn(4, C, L, generator=gen).cuda() * po.row_mask(4, L, valid, "cuda").float()
        res = torch.randn(4, C, L, generator=gen).cuda()
        lengths = torch.tensor(valid, dtype=torch.int32).cuda()
        y, hi, lo, _ = _run_pair(gens, kind, i, x, res=res, out16="hilo", lengths=lengths)
        ref, bound = _pair_ref(gens, kind, i, x, res=res, valid=valid)
        r = po.worst_ratio(y, ref, bound)
        WORST[sig] = max(WORST.get(sig, 0.0), r)
        if not r <= 1.0:
            failures.append((sig, "ragged", r))
        _check_planes(y, hi, lo, valid, (sig, "ragged planes"))
    assert not failures, failures


def test_pairs_persistent_loops(gens):
    """one pair per kernel instance at a length with more than 2 x (SM count) work items: every CTA runs several items, reusing
    its mid buffer and (streamed weights) cycling the ring through many phases"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    done = set()
    gen = torch.Generator().manual_seed(12)
    for kind, i, key, p in _pair_cases(gens):
        if p["kernel"] in done:
            continue
        done.add(p["kernel"])
        C = key[0]
        L = (2 * sms + 7) * p["pair_rows_item"] + 3
        x = torch.randn(1, C, L, generator=gen).cuda()
        res = torch.randn(1, C, L, generator=gen).cuda()
        y, _, _, ln = _run_pair(gens, kind, i, x, res=res, res_kind="f16")
        assert ln[0]["n_work"] > 2 * ln[0]["grid"], ln
        ref, bound = _pair_ref(gens, kind, i, x, res=res, res_kind="f16")
        _check(y, ref, bound, (kind, key, "persistent"), (kind, i) + key)
    assert len(done) == 4


EPI_VARIANTS = [dict(mode=m, red_add=r) for m in ("store", "add", "add_div") for r in (False, True)] + \
               [dict(mode="store", res_kind=k, out16="hilo") for k in ("f32", "f16", "hilo")] + \
               [dict(mode="add_div", res_kind="hilo", out16="f16"), dict(mode="add", res_kind="f16", out16="f16")]


def _variant_inputs(gen, B, C, L, valid, v):
    x = torch.randn(B, C, L, generator=gen).cuda() * po.row_mask(B, L, valid, "cuda").float()
    res = torch.randn(B, C, L, generator=gen).cuda()
    S = (torch.randn(B, C, L, generator=gen).cuda() * po.row_mask(B, L, valid, "cuda").float()) if v["mode"] != "store" else None
    return x, res, S


@pytest.mark.parametrize("v", EPI_VARIANTS, ids=lambda v: "-".join(f"{k}={v[k]}" for k in sorted(v)))
def test_pair_epilogue_variants(gens, v):
    """each pair kernel instance with every accumulate mode (red_add on / off), residual kind and fp16 output plane, ragged"""
    gen = torch.Generator().manual_seed(13)
    done = set()
    for kind, i, key, p in _pair_cases(gens):
        if p["kernel"] in done:
            continue
        done.add(p["kernel"])
        C, k, _ = key
        ri_ = p["pair_rows_item"]
        L, valid = ri_ + 37, [ri_ + 37, ri_ + 1]
        x, res, S = _variant_inputs(gen, 2, C, L, valid, v)
        lengths = torch.tensor(valid, dtype=torch.int32).cuda()
        rk = v.get("res_kind", "f32")
        y, hi, lo, ln = _run_pair(gens, kind, i, x, res=res, res_kind=rk, mode=v["mode"], red_add=v["red_add"] if "red_add" in v
                                  else False, S=S, out16=v.get("out16"), lengths=lengths)
        assert ln[0]["red_add"] == int(v.get("red_add", False) and v["mode"] == "add" and v.get("out16") is None), ln
        ref, bound = _pair_ref(gens, kind, i, x, res=res, res_kind=rk, mode=v["mode"], S=S, valid=valid)
        _check(y, ref, bound, (kind, key, v), (kind, i) + key)
        if v.get("out16"):
            _check_planes(y, hi, lo, valid, (kind, key, v))
    assert len(done) == 4


def test_pair_fused_vs_two_launches(gens):
    """the fused launch and c1 / c2 as two launches (what MB_TC_FUSE=0 runs) on identical inputs: both within the bound; whether
    they are bitwise equal is recorded (they need not be: the unfused c2 is a different kernel instance)"""
    gen = torch.Generator().manual_seed(14)
    failures = []
    for kind, i, key, p in _pair_cases(gens):
        C, k, _ = key
        L = 2 * p["pair_rows_item"] + (k - 1) // 2
        x = torch.randn(2, C, L, generator=gen).cuda()
        res = torch.randn(2, C, L, generator=gen).cuda()
        yf, _, _, _ = _run_pair(gens, kind, i, x, res=res)
        yu, _, _, ln = _run_pair(gens, kind, i, x, res=res, pair=2)
        assert len(ln) == 2 and ln[0]["kernel"][3] == 0 and ln[1]["kernel"][3] == 0, ln
        ref, bound = _pair_ref(gens, kind, i, x, res=res)
        sig = (kind, i) + key
        BITWISE[sig] = bool(torch.equal(yf, yu))
        for name, y in (("fused", yf), ("two launches", yu)):
            r = po.worst_ratio(y, ref, bound)
            WORST[sig] = max(WORST.get(sig, 0.0), r)
            if not r <= 1.0:
                failures.append((sig, name, r))
    print("fused == two launches bitwise:", BITWISE)
    assert not failures, failures


def _single_cases(gens):
    """(generator, op index) of one layer per plain kernel instance: HiFi-GAN ups.0 (256, 3-term split), resblocks.3.convs2.0
    (128, residual), ups.2 / ups.3 (64 / 32, transposed, split), and the k = 5 config's C = 128 layer (<128, 1, 64>)"""
    out = []
    for kind, prefix in (("hifigan", "ups.0"), ("hifigan", "resblocks.3.convs2.0"), ("hifigan", "ups.2"), ("hifigan", "ups.3"),
                         ("k5", "resblocks.0.convs2.0")):
        g, _ = gens[kind]
        i = next(j for j in range(g.num_layers()) if g.layer_info(j).split()[1] == prefix)
        out.append((kind, i))
    return out


@pytest.mark.parametrize("v", EPI_VARIANTS, ids=lambda v: "-".join(f"{k}={v[k]}" for k in sorted(v)))
def test_single_layer_epilogue_variants(gens, v):
    gen = torch.Generator().manual_seed(15)
    for kind, i in _single_cases(gens):
        g, sd = gens[kind]
        name, d = _info(g, i)
        p = g.tc_plan_info(i)
        transposed = name.startswith("ups.")
        s = d["stride"] if transposed else 1
        Lin = 300
        vin = [Lin, 123]
        valid = [n * s for n in vin]
        B, Lout = 2, Lin * s
        x = torch.randn(B, d["cin"], Lin, generator=gen).cuda() * po.row_mask(B, Lin, vin, "cuda").float()
        res = torch.randn(B, d["cout"], Lout, generator=gen).cuda()
        S = (torch.randn(B, d["cout"], Lout, generator=gen).cuda() * po.row_mask(B, Lout, valid, "cuda").float()) \
            if v["mode"] != "store" else None
        rk = v.get("res_kind", "f32")
        y, hi, lo, ln = g.debug_launch(i, x, mode=v["mode"], div=3.0, red_add=v.get("red_add", False), y_init=S, residual=res,
                                       res_kind=rk, res_slope=SLOPE, out16=v.get("out16"), out_slope=SLOPE,
                                       lengths=torch.tensor(vin, dtype=torch.int32).cuda())
        RAN.update(l["kernel"] for l in ln)
        assert ln[0]["kernel"] == (d["cout"], p["mt"], p["kc"], 0), (name, ln, p)
        w, b = _weights(sd, name, d["cin"], d["cout"], transposed)
        ref = po.layer_reference(x, w, b, dil=d["dil"], stride=s, transposed=transposed, slope_in=SLOPE, rounded=not p["x3"],
                                 res=res, res_kind=rk, res_slope=SLOPE, mode=v["mode"], S=S, div=3.0, valid=valid)
        bound = po.TOL * ref.abs().max() * po.row_mask(B, Lout, valid, "cuda")
        _check(y, ref, bound, (kind, name, v))
        if v.get("out16"):
            _check_planes(y, hi, lo, valid, (kind, name, v))


def test_not_a_pair_is_rejected(gens):
    from mockingbird_b200 import _lib

    g, _ = gens["hifigan"]
    i = next(j for j in range(g.num_layers()) if g.layer_info(j).split()[1] == "resblocks.3.convs1.0")  # C = 128: unfused
    with pytest.raises(_lib.MbError, match="not a fused pair"):
        g.debug_launch(i, torch.zeros(1, 128, 8, device="cuda"), pair=1)


def test_zz_every_kernel_instance_ran():
    """every tc_conv_kernel instance gan_tc.cu compiles was launched by a test of this module (run the whole module)"""
    from test_gan_tc_plan import compiled_instances

    if not WORST:
        pytest.skip("run with the rest of the module")
    print("worst |y - ref| / bound per pair signature:", {k: round(v, 4) for k, v in sorted(WORST.items())})
    assert compiled_instances() - RAN == set(), sorted(compiled_instances() - RAN)
