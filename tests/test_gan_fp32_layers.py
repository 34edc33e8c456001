"""The FP32 tap-conv kernels (csrc/gan_fp32.cu) one launch at a time (mb_gan_debug_f32), and Fre-GAN's single tensor-core layers
(mb_gan_debug_launch), against the float64 references of oracle/gan_fp32_oracle.py; and CPU self-tests of those references.

FP32 kernels: every distinct op signature of HiFi-GAN 16 kHz, HiFi-GAN 24 kHz and Fre-GAN, on fp32 handles (NCL tensors, as the
fp32 forward runs them) and the FP32 ops of f16tc handles (blocked fp32 tensors and fp16 / hi-lo output planes, as the tensor-core
forward runs them), at input lengths 1, 63, 64, 65 and 300 rows around the 64-row tile, B = 3 with ragged lengths, in the epilogue
mode the plan gives each op.  Inputs, residuals and running sums past each row's length are NaN: the kernel must not read them
into a valid row, and every output row past a length must be exactly 0.  Bound: tc_pair_oracle.TOL x max |ref| (the kernel's fp32
summation order).  The fp16 planes must equal the kernel's own fp32 result rounded as the epilogue rounds, bit for bit, and the
Cout = 1 kernel variants must equal each other bit for bit.  The last GPU test runs every FP32 kernel instance on a case of its
own and checks that each one ran.
"""
import os

import pytest
import torch

import gan_fp32_oracle as fo
import gan_oracle as go
import hifigan24k_oracle as o24
import ref_init as ri
import tc_pair_oracle as po

gpu = pytest.mark.gpu
WORST = {}

CONFIGS = {"hifigan": ri.HIFIGAN_CONFIG_16K, "hifigan24k": ri.HIFIGAN_CONFIG_24K, "fregan": ri.FREGAN_CONFIG}
LENS = {1: [1, 1, 1], 63: [63, 62, 1], 64: [64, 63, 33], 65: [65, 64, 1], 300: [300, 65, 64]}
MODES = {0: "store", 1: "add", 2: "add_div"}
SLOPE = 0.1
_GENS = {}


def _gen(name, precision, ups_x3=1):
    key = (name, precision, ups_x3)
    if key not in _GENS:
        from mockingbird_b200.vocoder.fregan.models import FreGAN
        from mockingbird_b200.vocoder.hifigan.models import Generator

        cfg = CONFIGS[name]
        sd = ri.fregan_state_dict(cfg, 0) if name == "fregan" else ri.hifigan_state_dict(cfg, 0)
        sd = ri.rescale_variance_preserving(sd, 1.0)
        before = os.environ.get("MB_TC_UPS_X3")
        os.environ["MB_TC_UPS_X3"] = str(ups_x3)  # read when the handle is created
        try:
            g = (FreGAN if name == "fregan" else Generator)(cfg, precision=precision)
        finally:
            if before is None:
                del os.environ["MB_TC_UPS_X3"]
            else:
                os.environ["MB_TC_UPS_X3"] = before
        g.cuda()
        g.load_state_dict(sd)
        g.eval()
        g.remove_weight_norm()
        _GENS[key] = (g, sd)
    return _GENS[key]


def _ops(g):
    """[(index, "conv" | "add", name, {cin, cout, k, dil, stride, res, mode, ...})] of the plan"""
    out = []
    for i in range(g.num_layers()):
        s = g.layer_info(i).split()
        out.append((i, s[0], s[1], {k: int(v) for k, v in (t.split("=") for t in s[2:])}))
    return out


def _conv_kind(cfg_name, name):
    if name.startswith("res_output.") or (cfg_name == "hifigan24k" and name.startswith("ups.")):
        return "nearest"
    return "transposed" if name.startswith(("ups.", "cond_up.")) else "conv"


def _slope_in(name):
    if name.startswith(("conv_pre", "cond_up.", "res_output.")):
        return 1.0
    return 0.01 if name == "conv_post" else SLOPE


def _weights(sd, name, kind, cin, cout):
    """checkpoint tensors zero-padded to the plan's channel counts (Fre-GAN's 16-channel stage runs with 32 on the tensor-core
    path), and the checkpoint's output channel count"""
    w, b = sd[name + ".weight"].double(), sd[name + ".bias"].double()
    shape = (cin, cout, w.shape[2]) if kind == "transposed" else (cout, cin, w.shape[2])
    wp = torch.zeros(shape, dtype=torch.float64)
    wp[: w.shape[0], : w.shape[1]] = w
    bp = torch.zeros(cout, dtype=torch.float64)
    bp[: b.shape[0]] = b
    return wp.cuda(), bp.cuda(), b.shape[0]


def _ragged(gen, B, C, L, valid, c_real=None):
    """(finite tensor zero past each row's length, the same with NaN there); channels >= c_real are zero in both (padded
    channels are identically zero in the forward)"""
    x = torch.randn(B, C, L, generator=gen, dtype=torch.float64).cuda().float()
    m = po.row_mask(B, L, valid, "cuda").float()
    x = x * m
    if c_real is not None:
        x[:, c_real:] = 0
    xn = torch.where(m.bool().expand_as(x), x, torch.full_like(x, float("nan")))
    if c_real is not None:
        xn[:, c_real:] = torch.where(m.bool().expand(B, C - c_real, L), 0.0, float("nan"))
    return x, xn


def _check(tag, y, ref, valid_out, cout_real=None):
    """within the bound in every row < valid_out[b], and exactly 0 (not NaN) in every row past it"""
    B, C, L = ref.shape
    m = po.row_mask(B, L, valid_out, "cuda")
    r = po.worst_ratio(y, ref, po.TOL * ref.abs().max() * m)
    WORST[tag] = max(WORST.get(tag, 0.0), r)
    assert r <= 1.0, (tag, r)
    past = y[(m == 0).expand_as(y)]
    assert bool((past == 0).all()), (tag, "rows past a length", past[past != 0][:4].tolist())
    if cout_real is not None and cout_real < C:
        assert float(y[:, cout_real:].abs().max()) == 0.0, (tag, "padded channels")


def _check_planes(tag, y, hi, lo, slope, hilo):
    """the fp16 plane(s) equal the kernel's own fp32 result rounded as the epilogue stores it, bit for bit"""
    hi_ref, lo_ref = fo.tstore_planes(y, slope, hilo)
    assert torch.equal(hi, hi_ref), (tag, "hi", float((hi - hi_ref).abs().max()))
    if hilo:
        assert torch.equal(lo, lo_ref), (tag, "lo", float((lo - lo_ref).abs().max()))


def _fp32_cases(g, name, precision):
    """first op of every distinct FP32 signature: (index, kind, name, info, has_dst2)"""
    ops = _ops(g)
    names = {n for _, _, n, _ in ops}
    seen, out = set(), []
    for i, kind, lname, d in ops:
        if kind == "conv" and precision != "fp32" and g.tc_plan_info(i)["use_tc"]:
            continue
        dst2 = kind == "conv" and lname.startswith("cond_up.") and ("x+=" + lname) not in names
        key = (kind, _conv_kind(name, lname) if kind == "conv" else "add", lname == "conv_post", lname == "conv_pre", dst2,
               d["cin"], d["cout"], d["k"], d["dil"], d["stride"], d["res"], d["mode"],
               lname.split("+=")[0] if kind == "add" else lname.split(".")[0])
        if key in seen:
            continue
        seen.add(key)
        out.append((i, kind, lname, d, dst2))
    return out


def _run_conv(g, sd, name, precision, i, lname, d, dst2, L, gen, x_layout=None, post=None, vin=None):
    B = 3
    vin = vin or LENS[L]
    kind = _conv_kind(name, lname)
    u = d["stride"]
    Lout = L * u
    vout = [n * u for n in vin]
    w, b, cout_real = _weights(sd, lname, kind, d["cin"], d["cout"])
    cin_real = sd[lname + ".weight"].shape[0 if kind == "transposed" else 1]
    x, xn = _ragged(gen, B, d["cin"], L, vin, cin_real)
    res = y0 = y2_0 = None
    resn = y0n = y2n = None
    if d["res"]:
        res, resn = _ragged(gen, B, d["cout"], Lout, vout, cout_real)
    mode = MODES[d["mode"]]
    if mode != "store":
        y0, y0n = _ragged(gen, B, d["cout"], Lout, vout, cout_real)
    if dst2:
        y2_0, y2n = _ragged(gen, B, d["cout"], Lout, vout, cout_real)
    tc = precision != "fp32"
    if x_layout is None:
        x_layout = "ncl" if (lname == "conv_pre" or not tc) else "f32b"
    y_layout = "ncl" if (lname == "conv_post" or not tc) else "f32b"
    planes = tc and lname != "conv_post"
    out16 = ("f16", "hilo")[L % 2] if planes else None
    y2_out16 = ("hilo", "f16")[L % 2] if planes and dst2 else None
    ncomp = len(CONFIGS[name]["resblock_kernel_sizes"])
    y, hi, lo, y2, hi2, lo2, kern = g.debug_launch_f32(
        i, xn, mode=mode, div=float(ncomp), y_init=y0n, residual=resn, out16=out16, out_slope=SLOPE,
        lengths=torch.tensor(vin, dtype=torch.int32).cuda(), x_layout=x_layout, y_layout=y_layout, y2_init=y2n,
        y2_out16=y2_out16, y2_slope=SLOPE, post=post)
    ref, ref2 = fo.tapconv_reference(x, w, b, kind, dil=d["dil"], stride=u, slope_in=_slope_in(lname), x_f16=x_layout == "f16b",
                                     res=res, mode=mode, y0=y0, div=float(ncomp), tanh=lname == "conv_post", valid_in=vin,
                                     valid_out=vout, y2_0=y2_0)
    tag = f"{name}/{precision} {lname} {kern} x={x_layout}"
    _check(tag, y, ref, vout, cout_real)
    if out16:
        _check_planes(tag, y, hi, lo, SLOPE, out16 == "hilo")
    if dst2:
        _check(tag + " y2", y2, ref2, vout, cout_real)
        if y2_out16:
            _check_planes(tag + " y2", y2, hi2, lo2, SLOPE, y2_out16 == "hilo")
    return y, kern


def _run_add(g, name, precision, i, lname, d, L, gen):
    """dst32 += src32 (no lengths: the forward's adds run over whole planes); the fp16 plane of the f16tc forward"""
    B, C = 3, d["cout"]
    x = torch.randn(B, C, L, generator=gen, dtype=torch.float64).cuda().float()
    y0 = torch.randn(B, C, L, generator=gen, dtype=torch.float64).cuda().float()
    tc = precision != "fp32"
    out16 = ("f16", "hilo")[L % 2] if tc else None
    layout = "f32b" if tc else "ncl"
    y, hi, lo, _, _, _, kern = g.debug_launch_f32(i, x, y_init=y0, out16=out16, out_slope=SLOPE, x_layout=layout,
                                                  y_layout=layout)
    assert kern == ("add_dst16" if out16 else "add"), kern
    tag = f"{name}/{precision} {lname} {kern}"
    assert torch.equal(y, y0 + x), tag  # one fp32 add per element
    WORST[tag] = 0.0
    if out16:
        _check_planes(tag, y, hi, lo, SLOPE, out16 == "hilo")
    return kern


@gpu
@pytest.mark.parametrize("L", sorted(LENS))
@pytest.mark.parametrize("precision", ["fp32", "f16tc"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_fp32_ops(name, precision, L):
    """every distinct FP32 op of the plan against its float64 reference; on fp32 handles at L = 65 also with an fp16 input plane"""
    g, sd = _gen(name, precision)
    gen = torch.Generator().manual_seed(L)
    cases = _fp32_cases(g, name, precision)
    assert cases
    failures = []  # every op is run and every failing one named, not only the first
    for i, kind, lname, d, dst2 in cases:
        cin = d["cin"]
        layouts = [None]
        if kind == "conv" and precision == "fp32" and L == 65 and cin % 8 == 0 and (cin < 64 or cin % 64 == 0):
            layouts.append("f16b")
        for x_layout in layouts:
            try:
                if kind == "add":
                    _run_add(g, name, precision, i, lname, d, L, gen)
                else:
                    _run_conv(g, sd, name, precision, i, lname, d, dst2, L, gen, x_layout=x_layout)
            except AssertionError as e:
                failures.append(str(e))
    for tag in sorted(t for t in WORST if t.startswith(f"{name}/{precision} ")):
        print(f"L={L} {tag}: worst |y - ref| / bound = {WORST[tag]:.4f}")
    assert not failures, "\n".join(failures)


@gpu
@pytest.mark.parametrize("precision", ["fp32", "f16tc"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_conv_post_variants_bitwise(name, precision):
    """conv_post on every Cout = 1 kernel: rows 1 / 2 / 4 per thread on NCL and blocked input, and the shared-memory tile kernel
    on blocked input, each against the float64 reference and bit-identical to the others on the same input layout (1100 rows:
    three tile blocks of 512)"""
    g, sd = _gen(name, precision)
    i, lname, d = next((i, n, d) for i, k, n, d in _ops(g) if n == "conv_post")
    for L in (1, 65, 300, 1100):
        vin = LENS.get(L, [L, 513, 512])
        for layout, posts in (("ncl", (1, 2, 4, None)), ("f32b", (1, 2, 4, "tile", None)), ("f16b", (1, 2, 4))):
            outs = []
            for post in posts:
                y, kern = _run_conv(g, sd, name, precision, i, lname, d, False, L, torch.Generator().manual_seed(L), x_layout=layout,
                                    post=post, vin=vin)
                outs.append((kern, y))
            for kern, y in outs[1:]:
                assert torch.equal(y, outs[0][1]), (name, precision, L, layout, kern, outs[0][0])
    tags = sorted(t for t in WORST if t.startswith(f"{name}/{precision} conv_post"))
    for t in tags:
        print(f"{t}: worst |y - ref| / bound = {WORST[t]:.4f}")


def _fregan_tc_singles(g):
    """first tensor-core op of every distinct signature that the forward launches alone (not as part of a fused pair)"""
    seen, out = set(), []
    for i, kind, lname, d in _ops(g):
        if kind != "conv":
            continue
        p = g.tc_plan_info(i)
        if not p["use_tc"] or p["fuse_next"] or p["fused_prev"]:
            continue
        key = (lname.split(".")[0], d["cin"], d["cout"], d["k"], d["dil"], d["stride"], d["res"], d["mode"])
        if key not in seen:
            seen.add(key)
            out.append((i, lname, d, p))
    return out


@gpu
@pytest.mark.parametrize("L", [1, 65, 300])
@pytest.mark.parametrize("ups_x3", [1, 0])
def test_fregan_single_tc_layers(ups_x3, L):
    """Fre-GAN's tensor-core layers that run alone (ups.*, cond_up.1-3, res_output.1/.2 over an un-activated hi/lo plane, the
    single layers of the 16 -> 32 channel stage) with lengths: the 3-term split against the unrounded float64 op, plain fp16
    layers against fp16-rounded operands; padded channels exactly 0"""
    g, sd = _gen("fregan", "f16tc", ups_x3)
    gen = torch.Generator().manual_seed(50 + L)
    cases = _fregan_tc_singles(g)
    names = {lname.split(".")[0] for _, lname, _, _ in cases}
    assert {"ups", "cond_up", "res_output"} <= names, names
    B, vin = 3, LENS[L]
    for i, lname, d, p in cases:
        kind = _conv_kind("fregan", lname)
        if lname.startswith(("ups.", "cond_up.", "res_output.")):
            assert p["x3"] == ups_x3, (lname, p)
        u = d["stride"]
        Lout, vout = L * u, [n * u for n in vin]
        w, b, cout_real = _weights(sd, lname, kind, d["cin"], d["cout"])
        cin_real = sd[lname + ".weight"].shape[0 if kind == "transposed" else 1]
        x, _ = _ragged(gen, B, d["cin"], L, vin, cin_real)
        res = y0 = None
        if d["res"]:
            res, _ = _ragged(gen, B, d["cout"], Lout, vout, cout_real)
        mode = MODES[d["mode"]]
        if mode != "store":
            y0, _ = _ragged(gen, B, d["cout"], Lout, vout, cout_real)
        y, _, _, ln = g.debug_launch(i, x, mode=mode, div=3.0, y_init=y0, residual=res, res_kind="f32" if res is not None else None,
                                     lengths=torch.tensor(vin, dtype=torch.int32).cuda())
        assert ln[0]["kernel"] == (d["cout"], p["mt"], p["kc"], 0), (lname, ln, p)
        wr = w if p["x3"] else po.q16(w)
        ref, _ = fo.tapconv_reference(x, wr, b, kind, dil=d["dil"], stride=u, slope_in=_slope_in(lname), x_f16=not p["x3"], res=res,
                                      mode=mode, y0=y0, div=3.0, valid_in=vin, valid_out=vout)
        tag = f"fregan/f16tc tc {lname} {'x3' if p['x3'] else 'f16'}"
        _check(tag, y, ref, vout, cout_real)
        print(f"L={L} {tag}: worst |y - ref| / bound = {WORST[tag]:.4f}")


@gpu
def test_every_fp32_kernel_instance_runs():
    """every FP32 kernel instance runs, and passes, on a case of its own: conv_pre (tapconv_f32), conv_post on each Cout = 1
    kernel (Cin = 32 on HiFi-GAN, 16 on the fp32 Fre-GAN) and the add ops with and without an fp16 plane (Fre-GAN fp32 / f16tc)"""
    want = {"tapconv_f32", "cout1<1>", "cout1<2>", "cout1<4>", "post_tile<7,4>", "post_tile<7,8>", "add", "add_dst16"}
    ran = set()
    gen = torch.Generator().manual_seed(7)
    for name, precision in (("hifigan", "fp32"), ("fregan", "fp32"), ("fregan", "f16tc")):
        g, sd = _gen(name, precision)
        for i, kind, lname, d, dst2 in _fp32_cases(g, name, precision):
            if kind == "add":
                ran.add(_run_add(g, name, precision, i, lname, d, 65, gen))
            elif lname == "conv_pre":
                ran.add(_run_conv(g, sd, name, precision, i, lname, d, dst2, 65, gen)[1])
            elif lname == "conv_post":
                for post in (1, 2, 4, "tile"):
                    ran.add(_run_conv(g, sd, name, precision, i, lname, d, dst2, 65, gen, x_layout="f32b", post=post)[1])
    print("FP32 kernel instances run:", sorted(ran))
    assert want <= ran, sorted(want - ran)


# ---- CPU self-tests of the references ------------------------------------------------------------------------------------------

TINY = {
    "hifigan": dict(ri.HIFIGAN_CONFIG_16K, upsample_rates=[5, 2], upsample_kernel_sizes=[10, 4], upsample_initial_channel=16,
                    resblock_kernel_sizes=[3, 7], resblock_dilation_sizes=[[1, 3], [1, 5]]),
    "hifigan24k": dict(ri.HIFIGAN_CONFIG_24K, upsample_rates=[3, 2], upsample_kernel_sizes=[7, 5], upsample_initial_channel=16,
                       resblock_kernel_sizes=[3, 11], resblock_dilation_sizes=[[1, 7], [1, 3]]),
    "fregan": dict(ri.FREGAN_CONFIG, upsample_rates=[2, 2, 2, 2, 2], upsample_kernel_sizes=[4, 4, 4, 4, 4], upsample_initial_channel=64,
                   resblock_kernel_sizes=[3, 5], resblock_dilation_sizes=[[1, 3], [1, 3]]),
}


def _mrf_ops(sd, cfg, i, X):
    """one MRF stage as the plan lowers it: per resblock conv pairs with the residual in the second conv's epilogue, the last
    conv of resblock j accumulating into S (store / add / add_div by the number of resblocks)"""
    nk = len(cfg["resblock_kernel_sizes"])
    S = None
    for j, (k, dils) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
        base = f"resblocks.{i * nk + j}"
        mode = "store" if j == 0 else ("add_div" if j == nk - 1 else "add")
        cur = X
        for m, dil in enumerate(dils):
            last = m == len(dils) - 1
            t, _ = fo.tapconv_reference(cur, sd[f"{base}.convs1.{m}.weight"], sd[f"{base}.convs1.{m}.bias"], "conv", dil=dil,
                                        slope_in=SLOPE)
            cur, _ = fo.tapconv_reference(t, sd[f"{base}.convs2.{m}.weight"], sd[f"{base}.convs2.{m}.bias"], "conv", slope_in=SLOPE,
                                          res=cur, mode=mode if last else "store", y0=S, div=float(nk))
        S = cur
    return S


def _chain(name, sd, cfg, mel):
    """the whole generator as a chain of single-launch references, in the order and with the epilogues of the FP32 plan"""
    x, _ = fo.tapconv_reference(mel, sd["conv_pre.weight"], sd["conv_pre.bias"], "conv")
    rates = cfg["upsample_rates"]
    if name != "fregan":
        kind = "nearest" if name == "hifigan24k" else "transposed"
        for i, u in enumerate(rates):
            key = f"ups.{i}.1" if kind == "nearest" else f"ups.{i}"
            x, _ = fo.tapconv_reference(x, sd[key + ".weight"], sd[key + ".bias"], kind, stride=u, slope_in=SLOPE)
            x = _mrf_ops(sd, cfg, i, x)
        y, _ = fo.tapconv_reference(x, sd["conv_post.weight"], sd["conv_post.bias"], "conv", slope_in=0.01, tanh=True)
        return y
    cond_level = len(rates) - 4
    cond, output = mel, None
    for i, u in enumerate(rates):
        if i >= cond_level:  # cond_up.j with x += cond as its second destination
            j = i - cond_level
            cond, x = fo.tapconv_reference(cond, sd[f"cond_up.{j}.weight"], sd[f"cond_up.{j}.bias"], "transposed", stride=rates[i - 1],
                                           y2_0=x)
        if i > cond_level:
            j = i - cond_level - 1
            src = x if output is None else output
            output, _ = fo.tapconv_reference(src, sd[f"res_output.{j}.1.weight"], sd[f"res_output.{j}.1.bias"], "nearest", stride=u)
        x, _ = fo.tapconv_reference(x, sd[f"ups.{i}.weight"], sd[f"ups.{i}.bias"], "transposed", stride=u, slope_in=SLOPE)
        x = _mrf_ops(sd, cfg, i, x)
        if output is not None:
            output = output + x
    y, _ = fo.tapconv_reference(output, sd["conv_post.weight"], sd["conv_post.bias"], "conv", slope_in=0.01, tanh=True)
    return y


@pytest.mark.parametrize("name", sorted(TINY))
def test_reference_chain_equals_oracle(name):
    """the single-launch references, chained as the FP32 plan chains its ops, give the oracle's generator (float64 oracle; the
    references evaluate each activation in fp32, hence 1e-5)"""
    cfg = TINY[name]
    sd = ri.fregan_state_dict(cfg, 0) if name == "fregan" else ri.hifigan_state_dict(cfg, 0)
    sd = {k: v.double() for k, v in ri.rescale_variance_preserving(sd, 1.0).items()}
    mel = torch.rand(2, 80, 9, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 8 - 4
    with torch.no_grad():
        ref = (o24.hifigan24k_forward(sd, cfg, mel) if name == "hifigan24k" else
               go.fregan_forward(sd, cfg, mel) if name == "fregan" else go.hifigan_forward(sd, cfg, mel))
        got = _chain(name, sd, cfg, mel)
    assert got.shape == ref.shape
    e = go.rel_errors(got, ref)
    assert e["max_rel"] < 1e-5, e


@pytest.mark.parametrize("u,k", [(5, 11), (4, 9), (3, 7), (2, 5), (8, 17), (2, 1)])
def test_folded_reference_equals_interpolate_conv(u, k):
    """nearest upsample + Conv1d as folded slabs (what fold_slabs_kernel packs and the kernel reads) equals interpolate + conv"""
    gen = torch.Generator().manual_seed(u * 100 + k)
    a = torch.randn(2, 6, 13, generator=gen, dtype=torch.float64)
    w = torch.randn(5, 6, k, generator=gen, dtype=torch.float64)
    b = torch.randn(5, generator=gen, dtype=torch.float64)
    ref = torch.nn.functional.conv1d(o24.interpolate_nearest(a, u), w, b, padding=(k - 1) // 2)
    assert torch.allclose(fo.op_forward(a, w, b, "nearest", stride=u), ref, rtol=0, atol=1e-12)
    assert torch.allclose(fo.folded_forward(a, w, b, u), ref, rtol=0, atol=1e-12)
    assert torch.allclose(o24.folded_forward(a, w, b, u), ref, rtol=0, atol=1e-12)


def test_reference_epilogue_and_masks():
    """mode, residual, tanh, the length masks and the second destination, checked element by element against a direct
    evaluation; each mutation the GPU tests must catch moves the reference past the bound"""
    gen = torch.Generator().manual_seed(4)
    B, C, L = 3, 4, 10
    x = torch.randn(B, C, L, generator=gen, dtype=torch.float64)
    w = torch.randn(C, C, 3, generator=gen, dtype=torch.float64)
    b = torch.randn(C, generator=gen, dtype=torch.float64)
    res, y0, y2 = (torch.randn(B, C, L, generator=gen, dtype=torch.float64) for _ in range(3))
    vin = vout = [10, 7, 1]
    y, s = fo.tapconv_reference(x, w, b, "conv", slope_in=SLOPE, res=res, mode="add_div", y0=y0, div=3.0, tanh=True, valid_in=vin,
                                valid_out=vout, y2_0=y2)
    a = po.act32(x, SLOPE) * po.row_mask(B, L, vin, "cpu")
    v = torch.tanh((y0 + torch.nn.functional.conv1d(a, w, b, padding=1) + res) / 3.0)
    m = po.row_mask(B, L, vout, "cpu")
    assert torch.allclose(y, v * m, rtol=0, atol=1e-14) and torch.allclose(s, (y2 + v) * m, rtol=0, atol=1e-14)
    assert float(y[1, :, 7:].abs().max()) == 0 and float(s[2, :, 1:].abs().max()) == 0
    bound = po.TOL * y.abs().max() * m
    wrong = [
        fo.tapconv_reference(x, w, b, "conv", slope_in=SLOPE, res=res, mode="add", y0=y0, tanh=True, valid_in=vin, valid_out=vout)[0],
        fo.tapconv_reference(x, w, b, "conv", slope_in=SLOPE, res=res, mode="add_div", y0=y0, div=3.0, tanh=True, valid_in=vin,
                             valid_out=[11, 8, 2])[0][:, :, :L],
        fo.tapconv_reference(x, w, b, "conv", slope_in=SLOPE, res=res, mode="add_div", y0=y0, div=3.0, tanh=True,
                             valid_out=vout)[0],
    ]
    for z in wrong:
        assert po.worst_ratio(z, y, bound) > 1.0


def test_tstore_planes():
    """hi = fp16_rn(lrelu(v)), lo = fp16_rn(lrelu(v) - hi): hi + lo carries v to about 2^-22 relative (for normal fp16 values);
    plain planes are hi alone"""
    v = torch.tensor([1.0 + 2.0 ** -12, -3.0, 0.0, 65504.0, 1e-6, -2.0 ** -30], dtype=torch.float32)
    hi, lo = fo.tstore_planes(v, SLOPE, True)
    a = torch.where(v > 0, v, v * SLOPE)
    assert torch.equal(hi, a.half().float())
    assert hi[0] == 1.0 and lo[0] == 2.0 ** -12 and hi[1] == (torch.tensor(-0.3).half().float())
    r = torch.randn(10000, generator=torch.Generator().manual_seed(5)) * 10
    hi, lo = fo.tstore_planes(r, SLOPE, True)
    a = torch.where(r > 0, r, r * SLOPE).double()
    err = (hi.double() + lo.double() - a).abs()
    assert bool((err <= a.abs() * 2.0 ** -21 + 2.0 ** -25).all())  # (below 2^-14 both halves share the subnormal step 2^-24)
    assert fo.tstore_planes(r, SLOPE, False)[1] is None
