"""Host side of the GAN vocoder generators (HiFi-GAN, Fre-GAN) over the mb_gan_* C ABI.

Mirrors the reference's ``Generator`` / ``FreGAN`` module surface (hifigan/models.py:96-162,
fregan/generator.py:79-179): construct from an AttrDict-like ``h``, ``load_state_dict`` with the
checkpoint's ``weight_g`` / ``weight_v`` keys, ``eval()``, ``remove_weight_norm()``, ``to(device)``,
call with ``mel [B, 80, T]`` -> ``wav [B, 1, T*hop]``.  All arithmetic runs in the CUDA library.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from .. import _lib


def _cfg_get(h, key, default=None):
    if isinstance(h, dict):
        return h.get(key, default)
    return getattr(h, key, default)


def fold_weight_norm(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """``remove_weight_norm`` (hifigan/models.py:152-162): w = g * v / ||v|| with the norm over all
    dims but 0 (weight_norm's default dim=0: C_out for Conv1d, C_in for ConvTranspose1d).
    Load-time only, evaluated with torch ops on the tensors' own device."""
    out: Dict[str, torch.Tensor] = {}
    for k, v in sd.items():
        if k.endswith(".weight_g"):
            base = k[: -len(".weight_g")]
            wv = sd[base + ".weight_v"].float()
            norm = wv.reshape(wv.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (wv.dim() - 1)))
            out[base + ".weight"] = wv * (v.float() / norm)
        elif k.endswith(".weight_v"):
            continue
        else:
            out[k] = v
    return out


class GanGenerator:
    """Common implementation; subclasses set KIND."""

    KIND = _lib.MB_GAN_HIFIGAN

    def __init__(self, h, precision: str = "auto", top_k: int = 4):
        self.h = h
        # the reference's own rule (hifigan/models.py:107): at 24 kHz every upsampling layer is nearest upsample + Conv1d
        self.kind = self.KIND
        if self.KIND == _lib.MB_GAN_HIFIGAN and _cfg_get(h, "sampling_rate", 16000) == 24000:
            self.kind = _lib.MB_GAN_HIFIGAN_INTERP
        rates = list(_cfg_get(h, "upsample_rates"))
        kernels = list(_cfg_get(h, "upsample_kernel_sizes"))
        rks = list(_cfg_get(h, "resblock_kernel_sizes"))
        rds = [list(d) for d in _cfg_get(h, "resblock_dilation_sizes")]
        cfg = _lib.GanConfig()
        cfg.kind = self.kind
        cfg.num_mels = 80  # hifigan/models.py:99 hard-codes 80 input channels
        cfg.upsample_initial_channel = int(_cfg_get(h, "upsample_initial_channel"))
        cfg.num_upsamples = len(rates)
        for i, (u, k) in enumerate(zip(rates, kernels)):
            cfg.upsample_rates[i] = int(u)
            cfg.upsample_kernel_sizes[i] = int(k)
        cfg.num_kernels = len(rks)
        cfg.num_dilations = len(rds[0])
        for j, (k, d) in enumerate(zip(rks, rds)):
            cfg.resblock_kernel_sizes[j] = int(k)
            if len(d) != len(rds[0]):
                raise ValueError("resblock_dilation_sizes must be rectangular")
            for m, dd in enumerate(d):
                cfg.resblock_dilation_sizes[j][m] = int(dd)
        cfg.resblock_type = 1 if str(_cfg_get(h, "resblock")) == "1" else 2
        cfg.fregan_top_k = int(top_k)
        if precision != "auto" and precision not in _lib.PRECISIONS:
            raise ValueError(f"precision must be 'auto' or one of {sorted(_lib.PRECISIONS)}")
        # "auto" (the drop-in default): the fast tensor-core mode (f16tc) is used only if, for THIS checkpoint, it stays within
        # half the 1e-3 parity tolerance of the FP32-equivalent tensor-core mode (f16x3) on a probe batch; otherwise f16x3 is
        # kept.  Decided once when the weights are uploaded (see _calibrate); `precision` then names the selected mode.
        self.requested_precision = precision
        self.calibration: Optional[Dict[str, float]] = None
        self.precision = "f16tc" if precision == "auto" else precision
        cfg.precision = _lib.PRECISIONS[self.precision]
        self._cfg = cfg
        self.num_kernels = len(rks)
        self.num_upsamples = len(rates)
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_gan_create(C.byref(cfg), C.byref(self._handle)))
        self.hop = int(_lib.lib().mb_gan_hop(self._handle))
        self._state: Optional[Dict[str, torch.Tensor]] = None  # host-side copy of the checkpoint
        self._arena: Optional[torch.Tensor] = None
        self._workspace: Optional[torch.Tensor] = None
        self._device: Optional[torch.device] = None
        self._ready = False
        self.training = True

    # -- nn.Module-like surface ------------------------------------------------------------------
    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        self._state = {k: v.detach() for k, v in state_dict.items()}
        self._ready = False
        return self

    def state_dict(self) -> Dict[str, torch.Tensor]:
        return dict(self._state or {})

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        self.training = mode
        return self

    def to(self, device):
        self._device = torch.device(device)
        if self._device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 generators run on CUDA only (no CPU fallback)")
        self._ready = False
        return self

    def cuda(self):
        return self.to(_lib.require_cuda())

    def remove_weight_norm(self):
        """Fold weight-norm and upload/pack the weights (hifigan/inference.py:53)."""
        if self._state is None:
            raise _lib.MbError("load_state_dict must be called before remove_weight_norm")
        self._state = fold_weight_norm(self._state)
        self._upload()
        return self

    # -- weights ---------------------------------------------------------------------------------
    AUTO_TOLERANCE = 5e-4  # half the north-star's 1e-3: f16tc is selected only with a 2x margin on the probe

    def _set_precision(self, precision: str) -> None:
        """re-create the library handle for another precision (weights must be uploaded again)"""
        L = _lib.lib()
        if self._handle.value:
            L.mb_gan_destroy(self._handle)
        self.precision = precision
        self._cfg.precision = _lib.PRECISIONS[precision]
        self._handle = C.c_void_p()
        _lib.check(L.mb_gan_create(C.byref(self._cfg), C.byref(self._handle)))
        self._workspace = None
        self._ready = False

    def _calibrate(self) -> None:
        """precision='auto': run a seeded probe batch (mel ~ U[-4, 4], the synthesizer's range; private generator, the global
        RNG is not touched) through f16x3 and f16tc and keep f16tc only if max- and rms-relative deviation <= AUTO_TOLERANCE"""
        dev = self._device
        probe = (torch.rand(2, 80, 64, generator=torch.Generator().manual_seed(20260922)) * 8 - 4).to(dev)
        self._set_precision("f16x3")
        self._upload_weights()
        ref = self.forward(probe).double()
        self._set_precision("f16tc")
        self._upload_weights()
        got = self.forward(probe).double()
        d = got - ref
        scale = float(ref.abs().max())
        rms = float(ref.pow(2).mean().sqrt())
        max_rel = float(d.abs().max()) / scale if scale > 0 else 0.0
        rms_rel = float(d.pow(2).mean().sqrt()) / rms if rms > 0 else 0.0
        ok = max_rel <= self.AUTO_TOLERANCE and rms_rel <= self.AUTO_TOLERANCE
        self.calibration = {"max_rel": max_rel, "rms_rel": rms_rel, "tolerance": self.AUTO_TOLERANCE, "selected": "f16tc" if ok else "f16x3"}
        if not ok:
            self._set_precision("f16x3")
            self._upload_weights()

    def _upload(self):
        if self.requested_precision == "auto":
            self._device = self._device or _lib.require_cuda()
            self._calibrate()
        else:
            self._upload_weights()

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """the weight-norm-folded convolution weights and biases, as mb_gan_set_weight takes them"""
        return {k: v for k, v in fold_weight_norm(self._state).items() if k.endswith(".weight") or k.endswith(".bias")}

    def _upload_weights(self):
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("gan", self._handle, self.weights_for_upload(), self._device)
        self._ready = True

    def packed_arena(self) -> torch.Tensor:
        """The packed device weights as one uint8 tensor (what multi-GPU start-up broadcasts)."""
        if not self._ready:
            self._upload()
        return self._arena

    # -- forward ---------------------------------------------------------------------------------
    def _ensure_workspace(self, B: int, T: int) -> torch.Tensor:
        need = int(_lib.lib().mb_gan_workspace_bytes(self._handle, B, T)) + 256
        if self._workspace is None or self._workspace.numel() < need:
            self._workspace = torch.empty(need, dtype=torch.uint8, device=self._device)
        return self._workspace

    def forward(self, x: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """mel [B, 80, T] (cuda fp32) -> wav [B, 1, T*hop].  ``lengths`` (int32 [B], optional, an
        extension over the reference) gives valid frames per utterance for padded batches."""
        if not self._ready:
            if self._state is None:
                raise _lib.MbError("Generator has no weights: call load_state_dict first")
            self._upload()
        if x.device.type != "cuda":
            raise _lib.MbError("Generator.forward expects a CUDA tensor (no CPU fallback)")
        if x.dim() != 3 or x.shape[1] != 80:
            raise ValueError(f"expected mel of shape [B, 80, T], got {tuple(x.shape)}")
        x = x.to(torch.float32).contiguous()
        B, _, T = x.shape
        out = torch.empty(B, 1, T * self.hop, dtype=torch.float32, device=x.device)
        if B == 0 or T == 0:
            return out
        with torch.cuda.device(x.device):
            ws = self._ensure_workspace(B, T)
            lp = None
            if lengths is not None:
                lengths = lengths.to(device=x.device, dtype=torch.int32).contiguous()
                lp = C.c_void_p(lengths.data_ptr())
            stream = torch.cuda.current_stream(x.device).cuda_stream
            _lib.check(_lib.lib().mb_gan_forward(self._handle, C.c_void_p(x.data_ptr()), lp, B, T,
                                                 C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()),
                                                 ws.numel(), C.c_void_p(stream)))
        return out

    __call__ = forward

    # -- measurement hooks (bench.py roofline) ---------------------------------------------------
    def forward_profiled(self, x: torch.Tensor):
        """forward with CUDA events around every layer; returns (wav, [ms per layer])."""
        if not self._ready:
            self._upload()
        x = x.to(torch.float32).contiguous()
        B, _, T = x.shape
        out = torch.empty(B, 1, T * self.hop, dtype=torch.float32, device=x.device)
        n = self.num_layers()
        ms = (C.c_float * n)()
        with torch.cuda.device(x.device):
            ws = self._ensure_workspace(B, T)
            stream = torch.cuda.current_stream(x.device).cuda_stream
            _lib.check(_lib.lib().mb_gan_forward_profiled(self._handle, C.c_void_p(x.data_ptr()), None, B, T,
                                                          C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()),
                                                          ws.numel(), C.c_void_p(stream), ms))
        return out, list(ms)

    def layer_work(self, i: int, B: int, T: int):
        macs, nbytes = C.c_double(), C.c_double()
        _lib.check(_lib.lib().mb_gan_layer_work(self._handle, i, B, T, C.byref(macs), C.byref(nbytes)))
        return macs.value, nbytes.value

    # -- test hooks ------------------------------------------------------------------------------
    def num_layers(self) -> int:
        return int(_lib.lib().mb_gan_num_layers(self._handle))

    def layer_info(self, i: int) -> str:
        buf = C.create_string_buffer(256)
        _lib.check(_lib.lib().mb_gan_layer_info(self._handle, i, buf, 256))
        return buf.value.decode()

    def debug_layer(self, i: int, x: torch.Tensor, residual: Optional[torch.Tensor], out_rows: int) -> torch.Tensor:
        if not self._ready:
            self._upload()
        x = x.contiguous().float()
        B, _, L = x.shape
        info = self.layer_info(i)
        cout = int(info.split("cout=")[1].split()[0])
        y = torch.zeros(B, cout, out_rows, dtype=torch.float32, device=x.device)
        cin = x.shape[1]
        need = 2 * B * max(cin, 64) * (L + 96) * 2 + 2 * B * cout * out_rows * 4 + (1 << 20)  # hi/lo planes: 2x channels
        ws = torch.empty(need, dtype=torch.uint8, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        rp = C.c_void_p(residual.contiguous().data_ptr()) if residual is not None else None
        _lib.check(_lib.lib().mb_gan_debug_layer(self._handle, i, C.c_void_p(x.data_ptr()), rp, B, L,
                                                 C.c_void_p(y.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                 C.c_void_p(stream)))
        return y

    def tc_plan_info(self, i: int) -> Dict[str, object]:
        """how the tensor-core forward runs op i (mb_gan_tc_plan_info): {"name": ..., key: int, "kernel": (N, MT, CW, PAIR)}"""
        buf = C.create_string_buffer(512)
        _lib.check(_lib.lib().mb_gan_tc_plan_info(self._handle, i, buf, 512))
        return _parse_report(buf.value.decode())

    EPI_MODES = {"store": 0, "add": 1, "add_div": 2}
    RES_KINDS = {None: 0, "f32": 1, "f16": 2, "hilo": 3}
    OUT16_KINDS = {None: 0, "f16": 1, "hilo": 2}

    def debug_launch(self, i: int, x: torch.Tensor, *, pair: int = 0, mode: str = "store", div: float = 1.0,
                     red_add: bool = False, y_init: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
                     res_kind: Optional[str] = None, res_slope: float = 1.0, out16: Optional[str] = None,
                     out_slope: float = 1.0, lengths: Optional[torch.Tensor] = None):
        """one tensor-core launch of layer i, or of the fused pair (i, i + 1) (pair=1) or that pair as two launches (pair=2),
        through mb_gan_debug_launch.  x [B, Cin, L] (not activated), residual [B, Cout, L*stride], y_init the running sum of the
        accumulate modes, lengths int32 [B] in input rows.  Returns (y, y16_hi, y16_lo, launches): fp32 NCL tensors (the fp16
        ones None when not requested) and one dict per kernel launch ({"kernel": (N, MT, CW, PAIR), "rows_item": ...})."""
        if not self._ready:
            self._upload()
        x = x.contiguous().float()
        B, cin, L = x.shape
        last = self.layer_info(i + (1 if pair else 0))
        cout = int(last.split("cout=")[1].split()[0])
        stride = int(last.split("stride=")[1].split()[0]) if not pair else 1
        Lout = L * stride
        dev = x.device
        y = (y_init.contiguous().float().clone() if y_init is not None
             else torch.zeros(B, cout, Lout, dtype=torch.float32, device=dev))
        c16 = (max(2 * cout, 64) if out16 == "hilo" else cout)
        y16 = torch.zeros(B, c16, Lout, dtype=torch.float32, device=dev) if out16 else None
        res = residual.contiguous().float() if residual is not None else None
        lens = lengths.to(device=dev, dtype=torch.int32).contiguous() if lengths is not None else None
        spec = _lib.GanDebugSpec()
        spec.layer_index, spec.pair, spec.mode, spec.div = i, pair, self.EPI_MODES[mode], div
        spec.red_add = int(red_add)
        spec.res_kind, spec.res_slope = self.RES_KINDS[res_kind], res_slope
        spec.out16, spec.out_slope = self.OUT16_KINDS[out16], out_slope
        spec.batch, spec.frames_in = B, L
        spec.x = x.data_ptr()
        spec.residual = res.data_ptr() if res is not None else None
        spec.lengths = lens.data_ptr() if lens is not None else None
        spec.y = y.data_ptr()
        spec.y16 = y16.data_ptr() if y16 is not None else None
        plane = B * 2 * max(cin, cout, 64) * (max(L, Lout) + 88) * 4 + (128 << 10) + 2048  # >= any plane of the launch
        ws = torch.empty(6 * plane + (1 << 20), dtype=torch.uint8, device=dev)
        report = C.create_string_buffer(1024)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(_lib.lib().mb_gan_debug_launch(self._handle, C.byref(spec), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                  C.c_void_p(stream), report, 1024))
        launches = [_parse_report(line) for line in report.value.decode().splitlines() if line]
        hi = lo = None
        if y16 is not None:
            hi = y16[:, :cout]
            lo = y16[:, c16 // 2:c16 // 2 + cout] if out16 == "hilo" else None
        return y, hi, lo, launches

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_gan_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def _parse_report(text: str) -> Dict[str, object]:
    """"[name] key=int ... kernel=N,MT,CW,PAIR" -> dict"""
    out: Dict[str, object] = {}
    for tok in text.split():
        if "=" not in tok:
            out["name"] = tok
            continue
        k, v = tok.split("=", 1)
        out[k] = tuple(int(p) for p in v.split(",")) if "," in v else int(v)
    return out


_pinned: Dict[str, torch.Tensor] = {}
_D2H_PIECE = 1 << 18  # smallest D2H piece, elements (1 MiB)


def _pinned_buffer(name: str, numel: int, dtype=torch.float32) -> torch.Tensor:
    """grow-only pinned staging buffers (cudaHostAlloc per call costs more than the copies it serves)"""
    buf = _pinned.get(name)
    if buf is None or buf.numel() < numel:
        buf = torch.empty(max(numel, 1), dtype=dtype).pin_memory()
        _pinned[name] = buf
    return buf


def infer_waveforms_batched(generator, device, mels: Sequence[np.ndarray], batch_size: int = 32) -> List[np.ndarray]:
    """Shared body of hifigan / fregan ``infer_waveforms``: length-sorted padded batches, each result equal to the per-utterance
    call (padding is masked at every layer on the device).  All batches are enqueued back to back (pinned H2D -> forward -> pinned
    D2H) and the host waits once at the end.  Host work is kept off the critical path (tools/time_e2e_host.py, cfg 2): the mels are
    packed into the pinned staging with numpy slice assignments (0.30 -> 0.1 ms for 32 utterances), the lengths travel in a
    pinned block too, and the copy out of the (reused) staging buffer (0.39 ms for 6.5 MB) overlaps the D2H transfer piece by piece."""
    n_mels = 80  # hifigan/models.py:99, fregan/generator.py hard-code 80 mel channels
    order = sorted(range(len(mels)), key=lambda i: -mels[i].shape[1])
    out: List[Optional[np.ndarray]] = [None] * len(mels)
    hop = generator.hop
    batches = []
    n_in = n_out = n_len = 0
    for s in range(0, len(order), batch_size):
        idx = order[s:s + batch_size]
        tmax = max(mels[i].shape[1] for i in idx)
        batches.append((idx, tmax, n_in, n_out, n_len))
        n_in += len(idx) * n_mels * tmax
        n_out += len(idx) * tmax * hop
        n_len += len(idx)
    host_in = _pinned_buffer("in", n_in)
    host_out = _pinned_buffer("out", n_out)
    host_len = _pinned_buffer("len", n_len, torch.int32)
    in_np, len_np = host_in.numpy(), host_len.numpy()
    pieces = []
    for idx, tmax, o_in, o_out, o_len in batches:
        if tmax == 0:
            continue
        nb = len(idx)
        hin = in_np[o_in:o_in + nb * n_mels * tmax].reshape(nb, n_mels, tmax)
        lens = [mels[i].shape[1] for i in idx]
        if lens[-1] == tmax:  # (sorted: the last one is the shortest) equal lengths: one stacked copy
            np.stack([np.asarray(mels[i]) for i in idx], out=hin, casting="unsafe")
        else:
            for r, i in enumerate(idx):
                t = lens[r]
                hin[r, :, :t] = mels[i]
                if t < tmax:
                    hin[r, :, t:] = 0.0
        len_np[o_len:o_len + nb] = lens
        dev = host_in[o_in:o_in + nb * n_mels * tmax].view(nb, n_mels, tmax).to(device, non_blocking=True)
        dlen = host_len[o_len:o_len + nb].to(device, non_blocking=True)
        wav = generator(dev, lengths=dlen)
        # D2H in a few pieces, an event after each: the host copies piece i out of the (reused) staging buffer while piece
        # i + 1 is still on the wire
        flat = wav.view(-1)
        n = flat.numel()
        step = max(_D2H_PIECE, -(-n // 8))
        for a in range(0, n, step):
            b = min(n, a + step)
            host_out[o_out + a:o_out + b].copy_(flat[a:b], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(device))
            pieces.append((ev, o_out + a, o_out + b))
    # ONE pass out of the staging buffer into a block this call owns (single-threaded on purpose: a multi-threaded torch copy
    # spins up one OpenMP thread per visible core and stalls for milliseconds under a container CPU quota); results are views of it
    block = np.empty(n_out, np.float32)
    out_np = host_out.numpy()
    for ev, a, b in pieces:
        ev.synchronize()
        block[a:b] = out_np[a:b]
    for idx, tmax, o_in, o_out, o_len in batches:
        if tmax == 0:
            for i in idx:
                out[i] = np.zeros(0, np.float32)
            continue
        wav = block[o_out:o_out + len(idx) * tmax * hop].reshape(len(idx), tmax * hop)
        for r, i in enumerate(idx):
            out[i] = wav[r, : mels[i].shape[1] * hop]
    return out  # type: ignore[return-value]
