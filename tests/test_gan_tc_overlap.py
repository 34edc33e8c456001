"""GPU tests of the persistent item loop of tc_conv_kernel in the instances whose accumulators take <= 64 registers per thread
(MT x N / 2 <= 64): the ones with room for a second accumulator set, which would let an item's epilogue overlap the next item's
MMAs (measured slower, DESIGN.md 3.3), and which run their epilogue units in pairs with the global reads one unit ahead.  Launch by
launch (mb_gan_debug_launch), against the float64 references of oracle/tc_pair_oracle.py, at the edges of the item loop:

* CTAs that get 1, 2, 3 and many work items;
* a next item in another utterance, in another phase of a transposed conv (stride 2), or wholly past a ragged length;
* every epilogue mode;
* every utterance of a ragged batch bitwise equal to its own B = 1 launch: a row's output does not depend on the schedule.
"""
import pytest
import torch

import tc_pair_oracle as po
from test_gan_tc_pair import EPI_VARIANTS, K5_CONFIG, SLOPE, _info, _make, _pair_cases, _pair_ref, _weights

import ref_init as ri

pytestmark = pytest.mark.gpu


def _small_acc(kernel):
    """MT x N / 2 <= 64 accumulator registers per thread"""
    n, mt, _, _ = kernel
    return mt * n // 2 <= 64


@pytest.fixture(scope="module")
def gens():
    return {"hifigan": _make("hifigan", ri.HIFIGAN_CONFIG_16K), "fregan": _make("fregan", ri.FREGAN_CONFIG),
            "k5": _make("hifigan", K5_CONFIG), "hifigan_x3": _make("hifigan", ri.HIFIGAN_CONFIG_16K, "f16x3")}


@pytest.fixture(scope="module")
def cases(gens):
    """one launch per such kernel instance and weight plan: fused pairs with resident and with streamed c1 weights, and the
    first layer launched alone of every (instance, weights resident, transposed) signature of HiFi-GAN at f16tc and f16x3 and of
    the k = 5 config (ups.3: stride 2; f16x3: 3-term-split layers)"""
    out, seen = [], set()
    for kind, i, key, p in _pair_cases(gens):
        k = tuple(p["kernel"])
        if _small_acc(k) and (k, p["pair_resident"]) not in seen:
            seen.add((k, p["pair_resident"]))
            out.append(dict(kind=kind, i=i, pair=True, kernel=k, rows_item=p["pair_rows_item"], stride=1, cin=key[0], cout=key[0]))
    for kind in ("hifigan", "hifigan_x3", "k5"):
        g, _ = gens[kind]
        for i in range(g.num_layers()):
            if g.layer_info(i).startswith("add"):
                continue
            p = g.tc_plan_info(i)
            if not p["use_tc"]:
                continue
            name, d = _info(g, i)
            k = (d["cout"], p["mt"], p["kc"], 0)  # the layer launched alone (a fused pair's convs too)
            if not _small_acc(k):
                continue
            stride = d["stride"] if name.startswith("ups.") else 1
            if (k, p["resident"], stride) in seen:
                continue
            seen.add((k, p["resident"], stride))
            out.append(dict(kind=kind, i=i, pair=False, kernel=k, rows_item=p["mt"] * 128, stride=stride, cin=d["cin"],
                            cout=d["cout"], name=name, x3=p["x3"]))
    assert {c["kernel"] for c in out} == {(64, 2, 64, 1), (64, 1, 64, 1), (32, 4, 32, 1), (64, 2, 64, 0), (32, 4, 64, 0),
                                          (128, 1, 64, 0)}, [(c["kind"], c["i"], c["kernel"]) for c in out]
    return out


def _inputs(gen, c, B, Lin, vin, v):
    s = c["stride"]
    valid = [n * s for n in vin]
    Lout = Lin * s
    x = torch.randn(B, c["cin"], Lin, generator=gen).cuda() * po.row_mask(B, Lin, vin, "cuda").float()
    res = torch.randn(B, c["cout"], Lout, generator=gen).cuda()
    S = (torch.randn(B, c["cout"], Lout, generator=gen).cuda() * po.row_mask(B, Lout, valid, "cuda").float()) \
        if v["mode"] != "store" else None
    return x, res, S, valid


def _launch(gens, c, x, res, S, v, vin):
    g, _ = gens[c["kind"]]
    y, hi, lo, ln = g.debug_launch(c["i"], x, pair=1 if c["pair"] else 0, mode=v["mode"], div=3.0, red_add=v.get("red_add", False),
                                   y_init=S, residual=res, res_kind=v.get("res_kind", "f32"), res_slope=SLOPE, out16=v.get("out16"),
                                   out_slope=SLOPE, lengths=torch.tensor(vin, dtype=torch.int32).cuda())
    assert len(ln) == 1 and tuple(ln[0]["kernel"]) == c["kernel"] and ln[0]["rows_item"] == c["rows_item"], (c, ln)
    return y, hi, lo, ln[0]


def _ratio(gens, c, x, res, S, v, valid, y):
    rk = v.get("res_kind", "f32")
    if c["pair"]:
        ref, bound = _pair_ref(gens, c["kind"], c["i"], x, res=res, res_kind=rk, mode=v["mode"], S=S, valid=valid)
    else:
        _, sd = gens[c["kind"]]
        _, d = _info(gens[c["kind"]][0], c["i"])
        transposed = c["name"].startswith("ups.")
        w, b = _weights(sd, c["name"], c["cin"], c["cout"], transposed)
        ref = po.layer_reference(x, w, b, dil=d["dil"], stride=c["stride"], transposed=transposed, slope_in=SLOPE,
                                 rounded=not c["x3"], res=res, res_kind=rk, res_slope=SLOPE, mode=v["mode"], S=S, div=3.0,
                                 valid=valid)
        B, _, L = ref.shape
        bound = po.TOL * ref.abs().max() * po.row_mask(B, L, valid, "cuda")
    return po.worst_ratio(y, ref, bound)


def test_items_per_cta(gens, cases):
    """B = 1 at lengths whose work items give every CTA 1 item, one CTA 2 items, one CTA 3 items, most CTAs 3 items and every CTA
    at least 5 items; the last item ends 5 rows short of its tile"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator().manual_seed(21)
    v = dict(mode="store")
    failures = []
    for c in cases:
        s, ri_ = c["stride"], c["rows_item"]
        most = set()  # items of the busiest CTA, per launch
        for n_work in (sms - 1, sms + 1, 2 * sms + 1, 3 * sms - 1, 5 * sms + 3):
            Lin = -(-n_work // s) * ri_ - 5
            x, res, S, valid = _inputs(gen, c, 1, Lin, [Lin], v)
            y, _, _, ln = _launch(gens, c, x, res, S, v, [Lin])
            most.add(-(-ln["n_work"] // ln["grid"]))
            r = _ratio(gens, c, x, res, S, v, valid, y)
            if not r <= 1.0:
                failures.append((c["kernel"], c["kind"], c["i"], n_work, r))
        assert {1, 2, 3} <= most and max(most) >= 5, (c["kernel"], most)
    assert not failures, failures


@pytest.mark.parametrize("v", EPI_VARIANTS, ids=lambda v: "-".join(f"{k}={v[k]}" for k in sorted(v)))
def test_ragged_batch_schedule_free(gens, cases, v):
    """a ragged batch of three utterances with about three items per CTA: a CTA's next item is often in the next utterance, and the
    third utterance (7 rows) leaves items wholly past its length.  Within the bound of the float64 reference, and every utterance
    bitwise equal to its own B = 1 launch (other CTAs, other neighbours in the pipeline)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator().manual_seed(22)
    failures = []
    for c in cases:
        s, ri_ = c["stride"], c["rows_item"]
        tiles = max(2, -(-3 * sms // (3 * s)))  # ~ 3 items per CTA over the batch
        Lin = tiles * ri_ - 3
        vin = [Lin, (tiles // 2) * ri_ + 1, 7]
        x, res, S, valid = _inputs(gen, c, 3, Lin, vin, v)
        y, hi, lo, ln = _launch(gens, c, x, res, S, v, vin)
        assert ln["n_work"] > ln["grid"], (c["kernel"], ln)
        r = _ratio(gens, c, x, res, S, v, valid, y)
        if not r <= 1.0:
            failures.append((c["kernel"], c["kind"], c["i"], "ragged", r))
        for b in range(3):
            y1, hi1, lo1, _ = _launch(gens, c, x[b:b + 1], res[b:b + 1], S[b:b + 1] if S is not None else None, v, vin[b:b + 1])
            same = torch.equal(y1, y[b:b + 1])
            if hi is not None:
                same = same and torch.equal(hi1, hi[b:b + 1]) and (lo is None or torch.equal(lo1, lo[b:b + 1]))
            if not same:
                failures.append((c["kernel"], c["kind"], c["i"], "utterance", b, "differs from its B = 1 launch"))
    assert not failures, failures
