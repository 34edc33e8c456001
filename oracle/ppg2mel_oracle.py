"""CPU oracle of the voice-conversion mel decoder (TEST INFRASTRUCTURE, not product code).

torch-CPU fp32 restatement, against torch.nn.functional only, of
  MelDecoderMOLv2.inference          models/ppg2mel/__init__.py:166-192
  Decoder.inference / attend / decode models/ppg2mel/rnn_decoder_mol.py:187-207, :267-315
  DecoderPrenet (dropout ALWAYS on)  rnn_decoder_mol.py:10-21
  MOLAttention (eval)                models/ppg2mel/utils/mol_attention.py:57-122
  Postnet (eval)                     models/ppg2mel/utils/cnn_postnet.py:7-52
working from a flat state_dict, for one utterance (B = 1, as the reference's inference is called).  The PreNet keep
masks are INJECTED (``masks``: a list of (keep1 [256], keep2 [128]) bool pairs, one per decoder step), which is what
makes a float parity statement possible; oracle/make_golden_ppg2mel.py captures them from the live reference by
wrapping torch.nn.functional.dropout.  ``sigmoid`` may be replaced (the precision study perturbs it by ulps).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F


def _branch(x, sd, p):
    """Conv1d k1 -> LeakyReLU -> IN -> [Conv1d k4 s2 p1 -> LeakyReLU -> IN] x 2 on x [1, C, T]"""
    x = F.instance_norm(F.leaky_relu(F.conv1d(x, sd[p + ".0.weight"]), 0.1), eps=1e-5)
    for i in (3, 6):
        x = F.conv1d(x, sd[f"{p}.{i}.weight"], sd[f"{p}.{i}.bias"], 2, 1)
        x = F.instance_norm(F.leaky_relu(x, 0.1), eps=1e-5)
    return x


def encode(sd, ppg: torch.Tensor, lf0_uv: torch.Tensor, spk: torch.Tensor) -> torch.Tensor:
    """ppg [T,144], lf0_uv [T,2], spk [256] -> memory [T_enc, 256] (__init__.py:172-180)"""
    x = _branch(ppg.t().unsqueeze(0), sd, "bnf_prenet").transpose(1, 2)
    x = x + _branch(lf0_uv.t().unsqueeze(0), sd, "pitch_convs").transpose(1, 2)
    s = F.normalize(spk.unsqueeze(0)).unsqueeze(1).expand(-1, x.size(1), -1)
    return F.linear(torch.cat([x, s], dim=-1), sd["reduce_proj.weight"], sd["reduce_proj.bias"])[0]


def _lstm(x, h, c, sd, p):
    g = F.linear(x, sd[p + ".weight_ih"], sd[p + ".bias_ih"]) + F.linear(h, sd[p + ".weight_hh"], sd[p + ".bias_hh"])
    i, f, gg, o = g.chunk(4, 1)
    c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
    return torch.sigmoid(o) * torch.tanh(c), c


def mol_alpha(params: torch.Tensor, mu_prev: torch.Tensor, T_enc: int,
              sigmoid: Callable = torch.sigmoid) -> Tuple[torch.Tensor, torch.Tensor]:
    """mixture parameters [1, 15] -> (alpha [1, T_enc], mu [1, 5]) as mol_attention.py:79-108"""
    M = 5
    w = torch.softmax(params[:, :M], dim=-1) + 1e-5
    sigma = F.softplus(params[:, M:2 * M]) + 1e-5
    mu = mu_prev + F.softplus(params[:, 2 * M:])
    j = (torch.arange(0, T_enc + 2.0) + 0.5)[:T_enc + 1]
    phi = w.unsqueeze(-1) * (1 / (1 + sigmoid((mu.unsqueeze(-1) - j) / sigma.unsqueeze(-1))))
    a = torch.sum(phi, dim=1)
    a = a[:, 1:] - a[:, :-1]
    a[a == 0] = 1e-5
    return a, mu


def postnet(sd, mel: torch.Tensor) -> torch.Tensor:
    """mel [T, 80] -> mel + Postnet(mel) [T, 80] (eval: BatchNorm with running stats, dropout off)"""
    x = mel.t().unsqueeze(0)
    for i in range(5):
        p = f"postnet.convolutions.{i}"
        x = F.conv1d(x, sd[p + ".0.conv.weight"], sd[p + ".0.conv.bias"], 1, 2)
        x = F.batch_norm(x, sd[p + ".1.running_mean"], sd[p + ".1.running_var"], sd[p + ".1.weight"], sd[p + ".1.bias"],
                         False, 0.1, 1e-5)
        if i < 4:
            x = torch.tanh(x)
    return mel + x[0].t()


def inference(sd: Dict[str, torch.Tensor], ppg: torch.Tensor, lf0_uv: torch.Tensor, spk: torch.Tensor,
              masks: Optional[List[Tuple[torch.Tensor, torch.Tensor]]] = None, sigmoid: Callable = torch.sigmoid,
              generator: Optional[torch.Generator] = None) -> Dict[str, torch.Tensor]:
    """one utterance; returns mel [2n,80], mel_postnet [2n,80], alignments [n,T_enc], stop [n] (logits), steps n.
    Without ``masks`` the keep masks are drawn from ``generator`` (Bernoulli(0.5))."""
    sd = {k: v.float() for k, v in sd.items() if v.dtype.is_floating_point}
    with torch.no_grad():
        memory = encode(sd, ppg.float(), lf0_uv.float(), spk.float())
        T_enc = memory.size(0)
        max_step = T_enc * 4 // 2
        min_step = max_step - 5
        x = torch.zeros(1, 80)
        ah, ac = torch.zeros(1, 512), torch.zeros(1, 512)
        dh, dc = torch.zeros(1, 512), torch.zeros(1, 512)
        ctx = torch.zeros(1, 256)
        mu = torch.zeros(1, 5)
        mels, aligns, stops = [], [], []
        while True:
            n = len(mels)
            if masks is not None:
                k1, k2 = masks[n]
            else:
                k1 = torch.rand(256, generator=generator) < 0.5
                k2 = torch.rand(128, generator=generator) < 0.5
            x = F.relu(F.linear(x, sd["decoder.prenet.layers.0.linear_layer.weight"])) * (k1.float() * 2.0)
            x = F.relu(F.linear(x, sd["decoder.prenet.layers.1.linear_layer.weight"])) * (k2.float() * 2.0)
            ah, ac = _lstm(torch.cat((x, ctx), -1), ah, ac, sd, "decoder.attention_rnn")
            q = "decoder.attention_layer.query_layer"
            params = F.linear(F.relu(F.linear(ah, sd[q + ".0.weight"], sd[q + ".0.bias"])), sd[q + ".2.weight"],
                              sd[q + ".2.bias"])
            alpha, mu = mol_alpha(params, mu, T_enc, sigmoid)
            ctx = torch.bmm(alpha.unsqueeze(1), memory.unsqueeze(0)).squeeze(1)
            dh, dc = _lstm(torch.cat((ah, ctx), -1), dh, dc, sd, "decoder.decoder_rnn_layers.0")
            out = torch.cat((dh, ctx), dim=1)
            mel = F.linear(out, sd["decoder.linear_projection.linear_layer.weight"],
                           sd["decoder.linear_projection.linear_layer.bias"])
            stop = F.linear(out, sd["decoder.stop_layer.linear_layer.weight"], sd["decoder.stop_layer.linear_layer.bias"])
            mels.append(mel)
            aligns.append(alpha)
            stops.append(stop.reshape(()))
            if torch.sigmoid(stop) > 0.5 and len(mels) >= min_step:
                break
            if len(mels) >= max_step:
                break
            x = mel[:, -80:]
        mel = torch.cat(mels, 0).view(-1, 80)
        return {"mel": mel, "mel_postnet": postnet(sd, mel), "alignments": torch.cat(aligns, 0),
                "stop": torch.stack(stops), "steps": len(mels)}


def rel_errors(got: torch.Tensor, ref: torch.Tensor) -> Dict[str, float]:
    got, ref = got.double().cpu(), ref.double().cpu()
    d = got - ref
    return {"max_rel": float(d.abs().max() / ref.abs().max().clamp_min(1e-30)),
            "rms_rel": float(d.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-30))}
