"""fatchord ``WaveRNN`` on the H100 path (reference: models/vocoder/wavernn/models/fatchord_version.py:88-257).

Same constructor and ``generate(mels, batched, target, overlap, mu_law, progress_callback)`` surface.
The conditioning network and the whole sample loop run in the CUDA library (mb_wavernn_*); the host
keeps only what the reference also does on the host in float64 numpy: cross-fade/unfold, mu-law
decoding, de-emphasis and the fade-out (fatchord_version.py:236-253).

Sampling noise.  ``Categorical(p).sample()`` is ``argmax(p / q)`` with ``q = empty_like(p).exponential_(1)``
drawn from the global torch generator (SURVEY.md fact 5).  ``rng="torch"`` (default) continues exactly
that stream - two ``nn.GRUCell`` constructions, then 2 MT19937 draws per element in ATen's order - from the
generator's own state: a host thread of the library runs the Mersenne Twister ~50x faster than ATen's serial
``exponential_`` and the device applies ATen's ``-log1p(-u)`` (csrc/mt_stream.cu), so under
``torch.manual_seed(s)`` the integer samples equal the reference's CPU run at full kernel speed, and the
global generator is left in the state the reference would leave it in.  ``rng="torch_host"`` is the plain
replay (one ``exponential_([B,512])`` per step on the host; A/B reference for the fast path);
``rng="device"`` uses the library's counter-based generator (no host noise).
"""
from __future__ import annotations

import ctypes as C
import time
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from .... import _lib
from .. import hparams as hp

CHUNK = 100  # steps per kernel call == the reference's progress cadence (fatchord_version.py:232-234)


def fold_geometry(total_len: int, target: int, overlap: int):
    """fold_with_overlap (:314-336): number of folds and their start offsets (the zero padding past
    the end is produced on the device)."""
    num_folds = (total_len - overlap) // (target + overlap)
    extended_len = num_folds * (overlap + target) + overlap
    remaining = total_len - extended_len
    if remaining != 0:
        num_folds += 1
    return num_folds, np.arange(num_folds, dtype=np.int32) * (target + overlap)


def torch_cpu_generator_position():
    """(state[624] uint32, left, next) of the global torch CPU generator (at::mt19937 inside the legacy
    CPUGeneratorImplState layout: seed u64 @0, left i32 @8, seeded i32 @12, next u64 @16, state u64[624] @24)"""
    st = torch.get_rng_state().numpy()
    left = int(st[8:12].view(np.int32)[0])
    nxt = int(st[16:24].view(np.uint64)[0])
    state = np.ascontiguousarray(st[24:24 + 624 * 8].view(np.uint64).astype(np.uint32))
    return state, left, nxt


def set_torch_cpu_generator_position(state: np.ndarray, left: int, nxt: int) -> None:
    st = torch.get_rng_state().numpy().copy()
    st[8:12] = np.array([left], np.int32).view(np.uint8)
    st[16:24] = np.array([nxt], np.uint64).view(np.uint8)
    st[24:24 + 624 * 8] = state.astype(np.uint64).view(np.uint8)
    torch.set_rng_state(torch.from_numpy(st))


def xfade_and_unfold(y: np.ndarray, target: int, overlap: int) -> np.ndarray:
    """Equal-power cross-fade and overlap-add of the folds (:340-402), float64 like the reference."""
    num_folds, length = y.shape
    target = length - 2 * overlap
    total_len = num_folds * (target + overlap) + overlap
    silence_len = overlap // 2
    fade_len = overlap - silence_len
    t = np.linspace(-1, 1, fade_len, dtype=np.float64)
    fade_in = np.concatenate([np.zeros(silence_len, dtype=np.float64), np.sqrt(0.5 * (1 + t))])
    fade_out = np.concatenate([np.sqrt(0.5 * (1 - t)), np.zeros(silence_len, dtype=np.float64)])
    y[:, :overlap] *= fade_in
    y[:, -overlap:] *= fade_out
    unfolded = np.zeros(total_len, dtype=np.float64)
    for i in range(num_folds):
        start = i * (target + overlap)
        unfolded[start:start + target + 2 * overlap] += y[i]
    return unfolded


def decode_mu_law(y: np.ndarray, mu: int) -> np.ndarray:
    """wavernn/audio.py:102-107 with from_labels=False"""
    mu = mu - 1
    return np.sign(y) / mu * ((1 + mu) ** np.abs(y) - 1)


def de_emphasis(x: np.ndarray) -> np.ndarray:
    """wavernn/audio.py:92-93"""
    from scipy.signal import lfilter

    return lfilter([1], [1, -hp.preemphasis], x)


class WaveRNN:
    def __init__(self, rnn_dims, fc_dims, bits, pad, upsample_factors, feat_dims, compute_dims, res_out_dims,
                 res_blocks, hop_length, sample_rate, mode='RAW'):
        if mode != 'RAW':
            raise NotImplementedError("only voc_mode='RAW' (the reference default, wavernn/hparams.py:24) is built; "
                                      "the MOL sampler is out of scope")
        self.mode = mode
        self.pad = pad
        self.n_classes = 2 ** bits
        self.rnn_dims = rnn_dims
        self.aux_dims = res_out_dims // 4
        self.hop_length = hop_length
        self.sample_rate = sample_rate
        cfg = _lib.WaveRNNConfig()
        cfg.rnn_dims, cfg.fc_dims, cfg.bits, cfg.pad = rnn_dims, fc_dims, bits, pad
        cfg.num_upsample = len(upsample_factors)
        for i, s in enumerate(upsample_factors):
            cfg.upsample_factors[i] = int(s)
        cfg.feat_dims, cfg.compute_dims, cfg.res_out_dims, cfg.res_blocks = feat_dims, compute_dims, res_out_dims, res_blocks
        self._total_scale = int(np.prod(upsample_factors))
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_wavernn_create(C.byref(cfg), C.byref(self._handle)))
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena = None
        self._ws = None
        self._mt = None          # mb_mtstream handle (pinned ring + side stream), created at first use
        self._mt_words = 0
        self._device = None
        self._ready = False
        self.training = True
        self.rng = "torch"
        self.post = "device"     # "device": mb_wavernn_postprocess (float64 kernels); "host": the numpy restatement
        self.seed = 0
        self.step = torch.zeros(1).long()

    # -- nn.Module-like surface ------------------------------------------------------------------
    def load_state_dict(self, sd, strict: bool = True):
        self._state = {k: v.detach() for k, v in sd.items()}
        if "step" in self._state:
            self.step = self._state["step"].clone()
        self._ready = False
        return self

    def state_dict(self):
        return dict(self._state or {})

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        self.training = mode
        return self

    def cuda(self):
        self._device = _lib.require_cuda()
        self._ready = False
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 WaveRNN runs on CUDA only (no CPU fallback)")
        self._device = device
        self._ready = False
        return self

    def get_step(self):
        return self.step.data.item()

    def _upload(self):
        if self._state is None:
            raise _lib.MbError("WaveRNN has no weights: call load_state_dict first")
        dev = self._device or _lib.require_cuda()
        self._device = dev
        L = _lib.lib()
        nbytes = int(L.mb_wavernn_arena_bytes(self._handle))
        with torch.cuda.device(dev):
            self._arena = torch.zeros(nbytes + 256, dtype=torch.uint8, device=dev)
            base = (self._arena.data_ptr() + 255) // 256 * 256
            _lib.check(L.mb_wavernn_set_arena(self._handle, C.c_void_p(base), nbytes))
            stream = torch.cuda.current_stream(dev).cuda_stream
            keep = []
            for name, t in self._state.items():
                if name == "step" or name.endswith("num_batches_tracked"):
                    continue
                d = t.to(device=dev, dtype=torch.float32).contiguous()
                keep.append(d)
                dims = (C.c_int64 * max(1, d.dim()))(*d.shape)
                _lib.check(L.mb_wavernn_set_weight(self._handle, name.encode(), C.c_void_p(d.data_ptr()), dims, d.dim(),
                                                   C.c_void_p(stream)))
            _lib.check(L.mb_wavernn_finalize(self._handle, C.c_void_p(stream)))
            torch.cuda.current_stream(dev).synchronize()
        self._ready = True

    def packed_arena(self) -> torch.Tensor:
        if not self._ready:
            self._upload()
        return self._arena

    # -- generate --------------------------------------------------------------------------------
    def generate_indices(self, mels: torch.Tensor, batched: bool, target: int, overlap: int, progress_callback=None,
                         noise: Optional[torch.Tensor] = None, rows: Optional[Tuple[int, int]] = None) -> np.ndarray:
        """host copy of generate_indices_device()"""
        out = self.generate_indices_device(mels, batched, target, overlap, progress_callback, noise, rows)
        return out if isinstance(out, np.ndarray) else out.cpu().numpy()

    def generate_indices_device(self, mels: torch.Tensor, batched: bool, target: int, overlap: int, progress_callback=None,
                                noise: Optional[torch.Tensor] = None, rows: Optional[Tuple[int, int]] = None):
        """the device part of generate(): class indices int16 [folds, steps].  ``rows=(lo, hi)`` runs only the folds
        [lo, hi) of the utterance (fold sharding across GPUs): the noise stream is still the whole utterance's, each
        fold reads its own rows, so a fold's samples do not depend on the sharding."""
        if not self._ready:
            self._upload()
        L = _lib.lib()
        dev = self._device
        mel = mels[0].to(device=dev, dtype=torch.float32).contiguous()  # [80, T]
        T = int(mel.shape[1])
        total = T * self._total_scale
        if batched:
            B, starts = fold_geometry(total, target, overlap)
            steps = target + 2 * overlap
        else:
            B, starts, steps = 1, np.zeros(1, dtype=np.int32), total
        if B <= 0 or steps <= 0:
            return np.zeros((max(B, 0), max(steps, 0)), np.int16)
        B_all, row0 = B, 0  # the noise stream always covers all folds of the utterance
        if rows is not None:
            row0, hi = int(rows[0]), int(rows[1])
            if not (0 <= row0 <= hi <= B_all):
                raise ValueError(f"rows {rows} outside the {B_all} folds")
            starts, B = starts[row0:hi], hi - row0
            if B == 0:
                if noise is None and self.rng in ("torch", "torch_host"):
                    self._skip_noise(B_all, steps)
                return np.zeros((0, steps), np.int16)
        start_t = time.time()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            need = int(L.mb_wavernn_workspace_bytes(self._handle, T, B, steps)) + 256
            if self._ws is None or self._ws.numel() < need:
                self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            ws = self._ws
            _lib.check(L.mb_wavernn_condition(self._handle, C.c_void_p(mel.data_ptr()), T, C.c_void_p(ws.data_ptr()),
                                              ws.numel(), C.c_void_p(stream.cuda_stream)))
            out = torch.empty(B, steps, dtype=torch.int16, device=dev)
            starts_c = (C.c_int32 * B)(*[int(s) for s in starts])
            if self.rng not in ("torch", "torch_host", "device"):
                raise ValueError(f"rng must be 'torch', 'torch_host' or 'device', got {self.rng!r}")
            use_host_noise = noise is not None or self.rng in ("torch", "torch_host")
            use_mt = noise is None and self.rng == "torch"
            if use_host_noise and noise is None:
                # the reference constructs two GRUCells before the loop: they consume the global RNG
                # (fatchord_version.py:160-161, 265-271)
                nn.GRUCell(self.rnn_dims, self.rnn_dims)
                nn.GRUCell(self.rnn_dims + self.aux_dims, self.rnn_dims)
            per_step = B_all * self.n_classes
            bufs = [torch.empty(CHUNK, B_all, self.n_classes, dtype=torch.float32).pin_memory() for _ in range(2)] \
                if use_host_noise and noise is None and not use_mt else None
            dbufs = [torch.empty(CHUNK, B_all, self.n_classes, dtype=torch.float32, device=dev) for _ in range(2)] \
                if use_host_noise else None
            raw = [torch.empty(CHUNK * per_step * 2, dtype=torch.int32, device=dev) for _ in range(2)] if use_mt else None
            if use_mt:
                words = CHUNK * per_step * 2
                if self._mt is None or self._mt_words < words:
                    if self._mt is not None:
                        L.mb_mtstream_destroy(self._mt)
                    self._mt = C.c_void_p()
                    _lib.check(L.mb_mtstream_create(words, 3, C.byref(self._mt)))
                    self._mt_words = words
                g_state, g_left, g_next = torch_cpu_generator_position()
                _lib.check(L.mb_mtstream_begin(self._mt, g_state.ctypes.data, g_left, g_next, steps * per_step * 2, words))
            evs = [torch.cuda.Event(), torch.cuda.Event()]
            step0 = 0
            ci = 0
            try:
                while step0 < steps:
                    n = min(CHUNK, steps - step0)
                    nptr = None
                    if use_host_noise:
                        slot = ci & 1
                        if noise is not None:
                            dbufs[slot][:n].copy_(noise[step0:step0 + n].to(torch.float32), non_blocking=True)
                        elif use_mt:
                            _lib.check(L.mb_mtstream_next(self._mt, n * per_step, C.c_void_p(raw[slot].data_ptr()),
                                                          C.c_void_p(dbufs[slot].data_ptr()), C.c_void_p(stream.cuda_stream)))
                        else:
                            if ci >= 2:
                                evs[slot].synchronize()  # the H2D that last used this pinned buffer is done
                            hb = bufs[slot]
                            for j in range(n):
                                hb[j].exponential_(1)  # same draw order as Categorical.sample(), one per step
                            dbufs[slot][:n].copy_(hb[:n], non_blocking=True)
                            evs[slot].record(stream)
                        nptr = C.c_void_p(dbufs[slot].data_ptr())
                    _lib.check(L.mb_wavernn_generate_rows(self._handle, starts_c, B, steps, step0, n, nptr, B_all, row0,
                                                          C.c_uint64(self.seed), C.c_void_p(out.data_ptr()),
                                                          C.c_void_p(ws.data_ptr()), ws.numel(),
                                                          C.c_void_p(stream.cuda_stream)))
                    if use_mt:
                        _lib.check(L.mb_mtstream_consumed(self._mt, C.c_void_p(stream.cuda_stream)))
                    if progress_callback is not None:
                        gen_rate = (step0 + 1) / max(time.time() - start_t, 1e-9) * B / 1000
                        progress_callback(step0, steps, B, gen_rate)
                    step0 += n
                    ci += 1
            finally:
                if use_mt:
                    # the generator is left exactly where the reference's own generate() would leave it
                    left_c, next_c = C.c_int32(), C.c_int32()
                    _lib.check(L.mb_mtstream_finish(self._mt, g_state.ctypes.data, C.byref(left_c), C.byref(next_c)))
                    set_torch_cpu_generator_position(g_state, left_c.value, next_c.value)
        return out

    def _skip_noise(self, B_all: int, steps: int) -> None:
        """advance the global generator as a full generate() would (a rank that owns no fold of the utterance)"""
        nn.GRUCell(self.rnn_dims, self.rnn_dims)
        nn.GRUCell(self.rnn_dims + self.aux_dims, self.rnn_dims)
        state, left, nxt = torch_cpu_generator_position()
        n = steps * B_all * self.n_classes * 2
        scratch = np.empty(1 << 20, np.uint32)
        l, x = C.c_int32(left), C.c_int32(nxt)
        while n > 0:
            m = min(n, scratch.size)
            _lib.check(_lib.lib().mb_mt19937_fill(state.ctypes.data, C.byref(l), C.byref(x), scratch.ctypes.data, m))
            n -= m
        set_torch_cpu_generator_position(state, l.value, x.value)

    def postprocess(self, idx: np.ndarray, frames: int, batched: bool, target: int, overlap: int, mu_law: bool) -> np.ndarray:
        """class indices [folds, steps] -> waveform, the host float64 tail of generate() (:236-253)"""
        wave_len = (frames - 1) * self.hop_length
        output = (2 * idx.astype(np.float32) / np.float32(self.n_classes - 1.) - np.float32(1.)).astype(np.float64)
        output = xfade_and_unfold(output, target, overlap) if batched else output[0]
        if mu_law:
            output = decode_mu_law(output, self.n_classes)
        if hp.apply_preemphasis:
            output = de_emphasis(output)
        fade_out = np.linspace(1, 0, 20 * self.hop_length)
        output = output[:wave_len]
        output[-20 * self.hop_length:] *= fade_out
        return output

    def postprocess_device(self, idx: torch.Tensor, frames: int, batched: bool, target: int, overlap: int, mu_law: bool) -> np.ndarray:
        """the same tail on the device (csrc/wavernn_post.cu): int16 [folds, steps] (cuda) -> host float64 waveform"""
        L = _lib.lib()
        idx = idx.to(torch.int16).contiguous()  # row-major [folds, steps] (a numpy view may arrive transposed)
        folds, steps = int(idx.shape[0]), int(idx.shape[1])
        dev = idx.device
        total = folds * (target + overlap) + overlap if batched else steps
        wave_len = (frames - 1) * self.hop_length
        fade_len = 20 * self.hop_length
        if min(total, wave_len) < fade_len:  # the reference's `output[-fade:] *= fade_out` raises on such short outputs too
            return self.postprocess(idx.cpu().numpy(), frames, batched, target, overlap, mu_law)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            need = int(L.mb_wavernn_postprocess_workspace_bytes(folds, steps, int(batched), target, overlap))
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            out = torch.empty(min(total, max(wave_len, 0)), dtype=torch.float64, device=dev)
            n_out = C.c_int64()
            _lib.check(L.mb_wavernn_postprocess(C.c_void_p(idx.data_ptr()), folds, steps, int(batched), target, overlap,
                                                self.n_classes, int(bool(mu_law)), float(hp.preemphasis) if hp.apply_preemphasis else 0.0,
                                                wave_len, fade_len, C.c_void_p(out.data_ptr()), C.byref(n_out), C.c_void_p(ws.data_ptr()),
                                                ws.numel(), C.c_void_p(stream.cuda_stream)))
            return out[: n_out.value].cpu().numpy()

    def generate_sharded(self, mels, target, overlap, mu_law, progress_callback=None, dst: int = 0):
        """batched generate() of ONE utterance with its folds dealt contiguously across the ranks of the default process
        group (SURVEY.md 8e row 2: folds are independent rows, fatchord_version.py:178-185): every rank computes the
        (cheap) conditioning, runs its folds, the int16 indices are gathered on `dst` which cross-fades / unfolds /
        decodes.  Returns the waveform on `dst`, None elsewhere.  Same samples as the single-GPU call."""
        from .... import distributed as mbd

        mu_law = mu_law if self.mode == 'RAW' else False
        rank, ws = mbd.world()
        total = int(mels.size(-1)) * self._total_scale
        B, _ = fold_geometry(total, target, overlap)
        lo, hi = mbd.fold_range(B, rank, ws)
        self.eval()
        idx = self.generate_indices(mels, True, target, overlap, progress_callback, rows=(lo, hi))
        full = mbd.gather_fold_rows(idx, B, dst=dst, device=self._device)
        self.train()
        if rank != dst:
            return None
        return self.postprocess(full, int(mels.size(-1)), True, target, overlap, mu_law)

    def generate(self, mels, batched, target, overlap, mu_law, progress_callback=None):
        mu_law = mu_law if self.mode == 'RAW' else False
        progress_callback = progress_callback or self.gen_display
        self.eval()
        idx = self.generate_indices_device(mels, batched, target, overlap, progress_callback)
        # sample = 2 * idx.float() / (n_classes - 1.) - 1.  (float32, :226) then float64 (:238)
        if self.post == "device" and not isinstance(idx, np.ndarray) and idx.numel() > 0:
            output = self.postprocess_device(idx, int(mels.size(-1)), batched, target, overlap, mu_law)
        else:
            idx = idx if isinstance(idx, np.ndarray) else idx.cpu().numpy()
            output = self.postprocess(idx, int(mels.size(-1)), batched, target, overlap, mu_law)
        self.train()  # side effect kept (:255)
        return output

    def gen_display(self, i, seq_len, b_size, gen_rate):
        pbar_len = 16
        done = int(pbar_len * (i + 1) / max(seq_len, 1))
        bar = '█' * done + '░' * (pbar_len - done)
        print(f'\r| {bar} {i * b_size}/{seq_len * b_size} | Batch Size: {b_size} | Gen Rate: {gen_rate:.1f}kHz | ',
              end='', flush=True)

    def __del__(self):
        try:
            if getattr(self, "_mt", None) is not None and self._mt.value:
                _lib.lib().mb_mtstream_destroy(self._mt)
                self._mt = None
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_wavernn_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
