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

``mode='MOL'`` (hparams ``voc_mode``) samples a 10-component discretized mixture of logistics instead
(distribution.py:87-123): fc3 has 30 outputs, the float32 sample is both the output and the next input.  Its
noise is ATen's float ``uniform_(1e-5, 1 - 1e-5)``, one MT19937 word per element, per step ``B x 10`` mixture
uniforms and then ``B`` logistic uniforms; the three ``rng`` choices replay / continue / replace that stream
the same way.
"""
from __future__ import annotations

import ctypes as C
import time
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn

from .... import _lib
from .. import hparams as hp

CHUNK = 100  # steps per kernel call == the reference's progress cadence (fatchord_version.py:232-234)
MOL_MIX = 10       # mixture components of the MOL sampler (fc3: 10 logit_probs | 10 means | 10 log_scales)
MOL_UNIFORMS = 11  # uniforms per row and step: 10 for the mixture pick, 1 for the logistic draw


def fold_geometry(total_len: int, target: int, overlap: int):
    """fold_with_overlap (:314-336): number of folds and their start offsets (the zero padding past
    the end is produced on the device)."""
    num_folds = (total_len - overlap) // (target + overlap)
    extended_len = num_folds * (overlap + target) + overlap
    remaining = total_len - extended_len
    if remaining != 0:
        num_folds += 1
    return num_folds, np.arange(num_folds, dtype=np.int32) * (target + overlap)


class RowPlan:
    """Row table of one multi-utterance sample loop (``WaveRNN.generate_many``).  Every utterance contributes its folds
    (``batched``) or one row of ``hop * frames`` steps as adjacent rows; utterances are ordered longest rows first (ties:
    input order), so the rows alive at any step are a prefix of the table and a 64-row block of the kernel empties as
    soon as its last row ends.

    ``order``: input index of the k-th utterance in row order; ``row_utt`` (k, not the input index), ``row_start``,
    ``row_steps``, ``row_fold``: one entry per row; ``utt_row0[k]``, ``utt_rows[k]``, ``utt_steps[k]``: the k-th
    utterance's block."""

    def __init__(self, frames: Sequence[int], batched: bool, target: int, overlap: int, total_scale: int = 200):
        geo = []
        for T in frames:
            total = int(T) * total_scale
            if batched:
                B, starts = fold_geometry(total, target, overlap)
                steps = target + 2 * overlap
            else:
                B, starts, steps = 1, np.zeros(1, dtype=np.int32), total
            if T <= 0 or B <= 0 or steps <= 0:
                raise ValueError(f"an utterance of {T} frames has no row to generate")
            geo.append((B, starts, steps))
        self.order = sorted(range(len(geo)), key=lambda u: (-geo[u][2], u))
        self.frames = [int(frames[u]) for u in self.order]
        self.utt_rows = [geo[u][0] for u in self.order]
        self.utt_steps = [geo[u][2] for u in self.order]
        self.utt_row0 = [int(v) for v in np.concatenate([[0], np.cumsum(self.utt_rows)[:-1]])]
        self.rows = int(sum(self.utt_rows))
        self.max_steps = self.utt_steps[0]
        self.row_utt = np.repeat(np.arange(len(geo), dtype=np.int32), self.utt_rows)
        self.row_start = np.concatenate([geo[u][1] for u in self.order]).astype(np.int32)
        self.row_steps = np.repeat(np.asarray(self.utt_steps, np.int32), self.utt_rows)
        self.row_fold = np.concatenate([np.arange(b, dtype=np.int32) for b in self.utt_rows])

    def live(self, step0: int) -> Tuple[int, int]:
        """(utterances, rows) still running at step ``step0``"""
        k = int(np.searchsorted(-np.asarray(self.utt_steps), -step0, side="left"))  # utt_steps > step0
        return k, (self.utt_row0[k] if k < len(self.utt_rows) else self.rows)

    def chunks(self, chunk: int):
        """(step0, nsteps, live utterances, live rows) of every kernel call"""
        out = []
        for step0 in range(0, self.max_steps, chunk):
            k, r = self.live(step0)
            out.append((step0, min(chunk, self.max_steps - step0), k, r))
        return out


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
        if mode not in ('RAW', 'MOL'):
            raise ValueError(f"Unknown model mode value - {mode!r} (voc_mode is 'RAW' or 'MOL')")
        self.mode = mode
        self.pad = pad
        self.n_classes = 2 ** bits if mode == 'RAW' else 3 * MOL_MIX
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
        kind = _lib.MB_WAVERNN_RAW if mode == 'RAW' else _lib.MB_WAVERNN_MOL
        _lib.check(_lib.lib().mb_wavernn_create_mode(C.byref(cfg), kind, C.byref(self._handle)))
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
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("wavernn", self._handle, self.weights_for_upload(), self._device)
        self._ready = True

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """the checkpoint without its step counter and the BatchNorm batch counters"""
        return {k: v for k, v in self._state.items() if k != "step" and not k.endswith("num_batches_tracked")}

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
        if self.mode != 'RAW':
            raise ValueError("generate_indices_device samples class indices (mode 'RAW'); a MOL model samples floats: "
                             "generate_samples_device")
        return self._sample_loop(mels, batched, target, overlap, progress_callback, noise, rows)

    def generate_samples(self, mels: torch.Tensor, batched: bool, target: int, overlap: int, progress_callback=None,
                         noise: Optional[torch.Tensor] = None, rows: Optional[Tuple[int, int]] = None) -> np.ndarray:
        """host copy of generate_samples_device()"""
        out = self.generate_samples_device(mels, batched, target, overlap, progress_callback, noise, rows)
        return out if isinstance(out, np.ndarray) else out.cpu().numpy()

    def generate_samples_device(self, mels: torch.Tensor, batched: bool, target: int, overlap: int, progress_callback=None,
                                noise: Optional[torch.Tensor] = None, rows: Optional[Tuple[int, int]] = None):
        """the device part of generate() of a MOL model: float32 samples [folds, steps] in [-1, 1].  ``noise``: the
        uniforms [steps, 11 * folds] (per step all folds' 10 mixture uniforms, then their logistic uniforms); ``rows`` as
        in generate_indices_device."""
        if self.mode != 'MOL':
            raise ValueError("generate_samples_device is the MOL sampler; a RAW model samples class indices: "
                             "generate_indices_device")
        return self._sample_loop(mels, batched, target, overlap, progress_callback, noise, rows)

    def _noise_layout(self, B_all: int):
        """(elements per step, MT19937 words per element) of the sampler's noise"""
        return (B_all * self.n_classes, 2) if self.mode == 'RAW' else (B_all * MOL_UNIFORMS, 1)

    def _sample_loop(self, mels, batched, target, overlap, progress_callback, noise, rows):
        mol = self.mode == 'MOL'
        out_dtype, out_np = (torch.float32, np.float32) if mol else (torch.int16, np.int16)
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
            return np.zeros((max(B, 0), max(steps, 0)), out_np)
        B_all, row0 = B, 0  # the noise stream always covers all folds of the utterance
        if rows is not None:
            row0, hi = int(rows[0]), int(rows[1])
            if not (0 <= row0 <= hi <= B_all):
                raise ValueError(f"rows {rows} outside the {B_all} folds")
            starts, B = starts[row0:hi], hi - row0
            if B == 0:
                if noise is None and self.rng in ("torch", "torch_host"):
                    self._skip_noise(B_all, steps)
                return np.zeros((0, steps), out_np)
        start_t = time.time()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            need = int(L.mb_wavernn_workspace_bytes(self._handle, T, B, steps))
            _lib.workspace(need, dev, self)
            ws = self._ws
            _lib.check(L.mb_wavernn_condition(self._handle, C.c_void_p(mel.data_ptr()), T, C.c_void_p(ws.data_ptr()),
                                              ws.numel(), C.c_void_p(stream.cuda_stream)))
            out = torch.empty(B, steps, dtype=out_dtype, device=dev)
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
            per_step, wpe = self._noise_layout(B_all)
            bufs = [torch.empty(CHUNK, per_step, dtype=torch.float32).pin_memory() for _ in range(2)] \
                if use_host_noise and noise is None and not use_mt else None
            dbufs = [torch.empty(CHUNK, per_step, dtype=torch.float32, device=dev) for _ in range(2)] \
                if use_host_noise else None
            raw = [torch.empty(CHUNK * per_step * wpe, dtype=torch.int32, device=dev) for _ in range(2)] if use_mt else None
            mt_next = L.mb_mtstream_next_uniform if mol else L.mb_mtstream_next
            if use_mt:
                words = CHUNK * per_step * wpe
                if self._mt is None or self._mt_words < words:
                    if self._mt is not None:
                        L.mb_mtstream_destroy(self._mt)
                    self._mt = C.c_void_p()
                    _lib.check(L.mb_mtstream_create(words, 3, C.byref(self._mt)))
                    self._mt_words = words
                g_state, g_left, g_next = torch_cpu_generator_position()
                _lib.check(L.mb_mtstream_begin(self._mt, g_state.ctypes.data, g_left, g_next, steps * per_step * wpe, words))
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
                            dbufs[slot][:n].copy_(noise[step0:step0 + n].to(torch.float32).reshape(n, per_step), non_blocking=True)
                        elif use_mt:
                            _lib.check(mt_next(self._mt, n * per_step, C.c_void_p(raw[slot].data_ptr()),
                                               C.c_void_p(dbufs[slot].data_ptr()), C.c_void_p(stream.cuda_stream)))
                        else:
                            if ci >= 2:
                                evs[slot].synchronize()  # the H2D that last used this pinned buffer is done
                            hb = bufs[slot]
                            for j in range(n):
                                if mol:  # sample_from_discretized_mix_logistic: temp [1, B, 10], then u [1, B]
                                    hb[j][:B_all * MOL_MIX].uniform_(1e-5, 1.0 - 1e-5)
                                    hb[j][B_all * MOL_MIX:].uniform_(1e-5, 1.0 - 1e-5)
                                else:
                                    hb[j].exponential_(1)  # same draw order as Categorical.sample(), one per step
                            dbufs[slot][:n].copy_(hb[:n], non_blocking=True)
                            evs[slot].record(stream)
                        nptr = C.c_void_p(dbufs[slot].data_ptr())
                    gen = L.mb_wavernn_generate_rows_mol if mol else L.mb_wavernn_generate_rows
                    _lib.check(gen(self._handle, starts_c, B, steps, step0, n, nptr, B_all, row0, C.c_uint64(self.seed),
                                   C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
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

    def _skip_noise(self, B_all: int, steps: int, advance: bool = True):
        """advance the global generator as a full generate() would (a rank that owns no fold of the utterance); returns
        the position (state, left, next) at which that generate() starts to draw its noise.  ``advance=False`` stops
        there (after the two GRUCell constructions)."""
        nn.GRUCell(self.rnn_dims, self.rnn_dims)
        nn.GRUCell(self.rnn_dims + self.aux_dims, self.rnn_dims)
        state, left, nxt = torch_cpu_generator_position()
        begin = (state.copy(), left, nxt)
        if not advance:
            return begin
        per_step, wpe = self._noise_layout(B_all)
        n = steps * per_step * wpe
        scratch = np.empty(1 << 20, np.uint32)
        l, x = C.c_int32(left), C.c_int32(nxt)
        while n > 0:
            m = min(n, scratch.size)
            _lib.check(_lib.lib().mb_mt19937_fill(state.ctypes.data, C.byref(l), C.byref(x), scratch.ctypes.data, m))
            n -= m
        set_torch_cpu_generator_position(state, l.value, x.value)
        return begin

    def noise_starts(self, blocks: Sequence[Tuple[int, int]], seeds: Optional[Sequence[int]]):
        """Generator position at which each utterance's noise begins; ``blocks[u] = (rows, steps)`` in input order.
        ``seeds=None``: where ``[generate(m) for m in mels]`` would begin utterance u under the global generator's current
        state - the stream is walked once on the host, and the generator is left where that loop leaves it.  ``seeds``:
        the position after ``torch.manual_seed(seeds[u])`` and the two GRUCell constructions; the global generator is
        put back as it was."""
        if seeds is None:
            return [self._skip_noise(B, steps) for B, steps in blocks]
        if len(seeds) != len(blocks):
            raise ValueError(f"{len(seeds)} seeds for {len(blocks)} utterances")
        saved = torch.get_rng_state()
        try:
            pos = []
            for (B, steps), s in zip(blocks, seeds):
                torch.default_generator.manual_seed(int(s))  # the CPU generator only: the noise is drawn from it
                pos.append(self._skip_noise(B, steps, advance=False))
        finally:
            torch.set_rng_state(saved)
        return pos

    def generate_many_device(self, mels: Sequence[torch.Tensor], batched: bool, target: int, overlap: int,
                             seeds: Optional[Sequence[int]] = None, progress_callback=None,
                             noise: Optional[Sequence[torch.Tensor]] = None, prefill=None) -> List[torch.Tensor]:
        """The device part of generate_many(): for utterance u (input order) the int16 class indices (RAW) or float32
        samples (MOL) ``[folds_u, steps_u]`` that generate_indices_device / generate_samples_device return for it alone,
        all utterances sharing one sequence of sample-loop launches.  ``mels[u]``: ``[1, 80, T_u]`` or ``[80, T_u]``.
        ``noise[u]``: injected noise in the single call's layout (``[steps_u, folds_u, 512]`` / ``[steps_u, 11 * folds_u]``).
        ``seeds``: with ``rng="torch"`` see noise_starts(); with ``rng="device"`` the built-in generator's seed per
        utterance (default: ``self.seed`` for all).  ``prefill``: value the output buffer holds before the loop (tests:
        a row writes nothing past its own last step); the results are views of that ``[rows, max_steps]`` buffer."""
        mol = self.mode == 'MOL'
        if not self._ready:
            self._upload()
        if len(mels) == 0:
            return []
        if self.rng not in ("torch", "device"):
            raise ValueError(f"generate_many draws its noise with rng 'torch' or 'device', not {self.rng!r} "
                             "('torch_host' is the single-utterance replay)")
        L = _lib.lib()
        dev = self._device
        mel2d = [m.reshape(-1, m.shape[-1]).to(dtype=torch.float32) for m in mels]
        plan = RowPlan([int(m.shape[1]) for m in mel2d], batched, target, overlap, self._total_scale)
        U, rows, max_steps = len(mel2d), plan.rows, plan.max_steps
        if seeds is not None and len(seeds) != U:
            raise ValueError(f"{len(seeds)} seeds for {U} utterances")
        per_row, wpe = self._noise_layout(1)  # noise elements per row and step, MT19937 words per element
        use_mt = noise is None and self.rng == "torch"
        if use_mt:
            blocks = [None] * U
            for k, u in enumerate(plan.order):
                blocks[u] = (plan.utt_rows[k], plan.utt_steps[k])
            starts = self.noise_starts(blocks, seeds)
            mt_state = np.stack([starts[u][0] for u in plan.order]).astype(np.uint32)
            mt_left = np.array([starts[u][1] for u in plan.order], np.int32)
            mt_next = np.array([starts[u][2] for u in plan.order], np.int32)
            wps = np.array([b * per_row * wpe for b in plan.utt_rows], np.uint64)
            col = np.concatenate([[0], np.cumsum(wps)[:-1]]).astype(np.uint64)
            threads = max(1, min(8, os.cpu_count() or 1))
        useed = [int(s) for s in seeds] if seeds is not None else [int(self.seed)] * U
        seeds_c = (C.c_uint64 * U)(*[useed[u] for u in plan.order])
        start_t = time.time()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            frames_c = (C.c_int32 * U)(*plan.frames)
            need = int(L.mb_wavernn_workspace_bytes_multi(self._handle, U, frames_c, rows, max_steps))
            if need == 0:
                raise _lib.MbError("generate_many: the utterances do not fit one loop (too many frames in all)")
            _lib.workspace(need, dev, self)
            ws = self._ws
            mel_cat = torch.cat([mel2d[u].reshape(-1) for u in plan.order]).to(dev).contiguous()
            _lib.check(L.mb_wavernn_condition_multi(self._handle, C.c_void_p(mel_cat.data_ptr()), frames_c, U,
                                                    C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(stream.cuda_stream)))
            out_dtype = torch.float32 if mol else torch.int16
            out = torch.empty(rows, max_steps, dtype=out_dtype, device=dev)
            if prefill is not None:
                out.fill_(prefill)
            as_i32 = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int32))
            row_utt, row_start, row_steps, row_fold = plan.row_utt, plan.row_start, plan.row_steps, plan.row_fold
            per_step = rows * per_row
            host_noise = noise is not None or use_mt
            dbufs = [torch.empty(CHUNK * per_step, dtype=torch.float32, device=dev) for _ in range(2)] if host_noise else None
            if use_mt:
                # chunk k+1 is drawn on the host and copied / converted on a side stream while the loop runs chunk k
                side = torch.cuda.Stream(dev)
                pinned = [torch.empty(CHUNK * per_step * wpe, dtype=torch.int32).pin_memory() for _ in range(2)]
                raw = [torch.empty(CHUNK * per_step * wpe, dtype=torch.int32, device=dev) for _ in range(2)]
                copied = [torch.cuda.Event() for _ in range(2)]
                consumed = [torch.cuda.Event() for _ in range(2)]
                convert = L.mb_mt_to_uniform if mol else L.mb_mt_to_exp
            gen = L.mb_wavernn_generate_multi_mol if mol else L.mb_wavernn_generate_multi
            for ci, (step0, n, k_live, n_live) in enumerate(plan.chunks(CHUNK)):
                nptr = None
                slot = ci & 1
                stride = n_live * per_row
                if noise is not None:
                    view = dbufs[slot][:n * stride].view(n, stride)
                    for k in range(k_live):
                        nk = min(n, plan.utt_steps[k] - step0)
                        c0, c1 = plan.utt_row0[k] * per_row, (plan.utt_row0[k] + plan.utt_rows[k]) * per_row
                        src = noise[plan.order[k]][step0:step0 + nk].to(torch.float32).reshape(nk, c1 - c0)
                        view[:nk, c0:c1].copy_(src, non_blocking=True)
                    nptr = C.c_void_p(dbufs[slot].data_ptr())
                elif use_mt:
                    if ci >= 2:
                        copied[slot].synchronize()  # the H2D that last read this pinned buffer is done
                    nst = np.minimum(n, np.asarray(plan.utt_steps[:k_live]) - step0).astype(np.int32)
                    _lib.check(L.mb_mt19937_fill_sources(k_live, mt_state.ctypes.data, mt_left.ctypes.data, mt_next.ctypes.data,
                                                         wps.ctypes.data, col.ctypes.data, nst.ctypes.data,
                                                         C.c_void_p(pinned[slot].data_ptr()), stride * wpe, threads))
                    with torch.cuda.stream(side):
                        if ci >= 2:
                            side.wait_event(consumed[slot])
                        raw[slot][:n * stride * wpe].copy_(pinned[slot][:n * stride * wpe], non_blocking=True)
                        copied[slot].record(side)
                        _lib.check(convert(C.c_void_p(raw[slot].data_ptr()), C.c_void_p(dbufs[slot].data_ptr()), n * stride,
                                           C.c_void_p(side.cuda_stream)))
                    stream.wait_stream(side)
                    nptr = C.c_void_p(dbufs[slot].data_ptr())
                _lib.check(gen(self._handle, as_i32(row_utt), as_i32(row_start), as_i32(row_steps), as_i32(row_fold), rows,
                               seeds_c, max_steps, step0, n, n_live, nptr, C.c_void_p(out.data_ptr()),
                               C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(stream.cuda_stream)))
                if use_mt:
                    consumed[slot].record(stream)
                if progress_callback is not None:
                    gen_rate = (step0 + 1) / max(time.time() - start_t, 1e-9) * n_live / 1000
                    progress_callback(step0, max_steps, n_live, gen_rate)
            if use_mt:
                stream.synchronize()  # the pinned and raw buffers die with this frame
        res = [None] * U
        for k, u in enumerate(plan.order):
            r0 = plan.utt_row0[k]
            res[u] = out[r0:r0 + plan.utt_rows[k], :plan.utt_steps[k]]
        return res

    def generate_many(self, mels: Sequence[torch.Tensor], batched, target, overlap, mu_law, seeds=None,
                      progress_callback=None) -> List[np.ndarray]:
        """generate() for a list of utterances ``[1, 80, T_u]`` in one sample loop: the float64 waveforms in input order,
        each what ``generate(mels[u], ...)`` returns for it alone.  ``seeds=None``: as the Python loop of generate() calls
        under the global generator's state (which is left where that loop leaves it); ``seeds=[s_u]``: utterance u as
        under ``torch.manual_seed(s_u)``, the global generator untouched."""
        mu_law = mu_law if self.mode == 'RAW' else False
        fade = 20 * self.hop_length
        for m in mels:  # the single call fails on these in its fade-out, after generating
            T = int(m.shape[-1])
            total = T * self._total_scale
            span = fold_geometry(total, target, overlap)[0] * (target + overlap) + overlap if batched else total
            if min(span, (T - 1) * self.hop_length) < fade:
                raise ValueError(f"an utterance of {T} frames is shorter than the {fade}-sample fade-out")
        self.eval()
        idx = self.generate_many_device(mels, batched, target, overlap, seeds, progress_callback or self.gen_display)
        wavs = []
        for m, rows in zip(mels, idx):
            T = int(m.shape[-1])
            if self.post == "device":
                wavs.append(self.postprocess_device(rows, T, batched, target, overlap, mu_law))
            else:
                wavs.append(self.postprocess(rows.cpu().numpy(), T, batched, target, overlap, mu_law))
        self.train()  # side effect of generate() kept
        return wavs

    def postprocess(self, idx: np.ndarray, frames: int, batched: bool, target: int, overlap: int, mu_law: bool) -> np.ndarray:
        """class indices [folds, steps] (RAW) or float samples (MOL) -> waveform, the host float64 tail of generate()
        (:236-253)"""
        wave_len = (frames - 1) * self.hop_length
        if self.mode == 'MOL':
            output = idx.astype(np.float32).astype(np.float64)
        else:
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
        """the same tail on the device (csrc/wavernn_post.cu): int16 indices (RAW) or float32 samples (MOL) [folds, steps]
        (cuda) -> host float64 waveform"""
        L = _lib.lib()
        mol = self.mode == 'MOL'
        # row-major [folds, steps] (a numpy view may arrive transposed)
        idx = idx.to(torch.float32 if mol else torch.int16).contiguous()
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
            ws = _lib.workspace(need, dev)
            out = torch.empty(min(total, max(wave_len, 0)), dtype=torch.float64, device=dev)
            n_out = C.c_int64()
            preemph = float(hp.preemphasis) if hp.apply_preemphasis else 0.0
            if mol:
                _lib.check(L.mb_wavernn_postprocess_f32(C.c_void_p(idx.data_ptr()), folds, steps, int(batched), target, overlap,
                                                        preemph, wave_len, fade_len, C.c_void_p(out.data_ptr()), C.byref(n_out),
                                                        C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(stream.cuda_stream)))
                return out[: n_out.value].cpu().numpy()
            _lib.check(L.mb_wavernn_postprocess(C.c_void_p(idx.data_ptr()), folds, steps, int(batched), target, overlap,
                                                self.n_classes, int(bool(mu_law)), float(hp.preemphasis) if hp.apply_preemphasis else 0.0,
                                                wave_len, fade_len, C.c_void_p(out.data_ptr()), C.byref(n_out), C.c_void_p(ws.data_ptr()),
                                                ws.numel(), C.c_void_p(stream.cuda_stream)))
            return out[: n_out.value].cpu().numpy()

    def generate_sharded(self, mels, target, overlap, mu_law, progress_callback=None, dst: int = 0):
        """batched generate() of ONE utterance with its folds dealt contiguously across the ranks of the default process
        group (SURVEY.md 8e row 2: folds are independent rows, fatchord_version.py:178-185): every rank computes the
        (cheap) conditioning, runs its folds, the int16 indices (float32 samples for MOL) are gathered on `dst` which
        cross-fades / unfolds / decodes.  Returns the waveform on `dst`, None elsewhere.  Same samples as the single-GPU
        call."""
        from .... import distributed as mbd

        mu_law = mu_law if self.mode == 'RAW' else False
        rank, ws = mbd.world()
        total = int(mels.size(-1)) * self._total_scale
        B, _ = fold_geometry(total, target, overlap)
        lo, hi = mbd.fold_range(B, rank, ws)
        self.eval()
        run = self.generate_samples if self.mode == 'MOL' else self.generate_indices
        idx = run(mels, True, target, overlap, progress_callback, rows=(lo, hi))
        full = mbd.gather_fold_rows(idx, B, dst=dst, device=self._device)
        self.train()
        if rank != dst:
            return None
        return self.postprocess(full, int(mels.size(-1)), True, target, overlap, mu_law)

    def generate(self, mels, batched, target, overlap, mu_law, progress_callback=None):
        mu_law = mu_law if self.mode == 'RAW' else False
        progress_callback = progress_callback or self.gen_display
        self.eval()
        run = self.generate_samples_device if self.mode == 'MOL' else self.generate_indices_device
        idx = run(mels, batched, target, overlap, progress_callback)
        # RAW: sample = 2 * idx.float() / (n_classes - 1.) - 1.  (float32, :226) then float64 (:238); MOL: the float32 sample
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
