"""``Tacotron`` on the H100 path (reference: models/synthesizer/models/tacotron.py:140-298).

Same constructor arguments and ``generate(x, speaker_embedding, steps=2000, style_idx=0,
min_stop_token=5) -> (mel_outputs, linear, attn_scores)`` surface; ``r`` property backed by the loaded
``decoder.r`` buffer (base.py:16-22).  All layers run in the CUDA library (mb_tacotron_*).

The reference's PreNet dropout is always active (pre_net.py:23,26), so generate() is stochastic.
``dropout_masks=(enc, dec)`` injects keep-masks (uint8/bool, enc [2,B,Tc,256], dec [steps/r,2,B,256]) for
reproducible comparisons; otherwise they are drawn on the device from ``seed``.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from ... import _lib
from ..hparams import gst_hparams

# rows per ragged batch of generate_many (at most 128, the tensor-core decoder's limit); see DESIGN.md section 4b
MANY_CHUNK_ROWS = 128


def many_plan(lengths, chunk_rows):
    """generate_many's batches: utterance indices sorted longest first (ties in input order), cut into chunks of at most
    ``chunk_rows`` (1..128)"""
    if not 1 <= int(chunk_rows) <= 128:
        raise ValueError(f"chunk_rows must be in [1, 128], got {chunk_rows}")
    order = sorted(range(len(lengths)), key=lambda i: (-int(lengths[i]), i))
    return [order[k:k + int(chunk_rows)] for k in range(0, len(order), int(chunk_rows))]


class StreamSchedule:
    """The host side of ``Tacotron.generate_stream``: which text enters which slot, and when each batch of texts is encoded.

    Texts are admitted longest first, ties in input order (``many_plan``'s order), each into the lowest free slot.  They are
    encoded in batches of ``slots`` texts in that order into a staging pool of two halves of ``slots`` rows: batch k goes to
    half k % 2, so it can be encoded once every text of batch k - 2 has been admitted."""

    def __init__(self, lengths, slots):
        if not 1 <= int(slots) <= 128:
            raise ValueError(f"slots must be in [1, 128], got {slots}")
        self.slots = int(slots)
        self.order = [i for chunk in many_plan(lengths, self.slots) for i in chunk]
        self.batches = [self.order[k:k + self.slots] for k in range(0, len(self.order), self.slots)]
        self.free = list(range(self.slots))
        self.pos = 0      # texts admitted so far (a position in `order`)
        self.encoded = 0  # batches handed to the encoder so far

    def pool_row(self, q):
        """staging-pool row of the text at position q of the admission order"""
        return (q // self.slots) % 2 * self.slots + q % self.slots

    def to_encode(self):
        """batches whose pool half is free now: list of (pool row of the first text, texts)"""
        out = []
        while self.encoded < len(self.batches) and self.pos >= (self.encoded - 1) * self.slots:
            out.append((self.pool_row(self.encoded * self.slots), self.batches[self.encoded]))
            self.encoded += 1
        return out

    def admit(self):
        """texts for the free slots: list of (slot, text, pool row); only texts whose batch has been encoded"""
        out = []
        self.free.sort(reverse=True)
        while self.free and self.pos < len(self.order) and self.pos // self.slots < self.encoded:
            out.append((self.free.pop(), self.order[self.pos], self.pool_row(self.pos)))
            self.pos += 1
        return out

    def finish(self, slot):
        self.free.append(int(slot))

    def busy(self):
        return self.slots - len(self.free)

    def done(self):
        return self.pos == len(self.order) and not self.busy()


class Tacotron:
    def __init__(self, embed_dims, num_chars, encoder_dims, decoder_dims, n_mels, fft_bins, postnet_dims, encoder_K,
                 lstm_dims, postnet_K, num_highways, dropout, stop_threshold, speaker_embedding_size):
        if fft_bins != n_mels:
            raise NotImplementedError("post_proj to fft_bins != n_mels is not part of the inference path")
        if abs(dropout - 0.5) > 1e-9:
            raise NotImplementedError("PreNet dropout p must be 0.5 (hparams.tts_dropout)")
        cfg = _lib.TacotronConfig()
        cfg.num_chars, cfg.embed_dims, cfg.encoder_dims, cfg.decoder_dims = num_chars, embed_dims, encoder_dims, decoder_dims
        cfg.n_mels, cfg.postnet_dims, cfg.encoder_K, cfg.lstm_dims = n_mels, postnet_dims, encoder_K, lstm_dims
        cfg.postnet_K, cfg.num_highways, cfg.speaker_embedding_size = postnet_K, num_highways, speaker_embedding_size
        cfg.gst_E, cfg.gst_tokens, cfg.gst_heads, cfg.max_r = gst_hparams.E, gst_hparams.token_num, gst_hparams.num_heads, 20
        self._cfg = cfg
        self.n_mels = n_mels
        self.encoder_dims, self.decoder_dims, self.lstm_dims = encoder_dims, decoder_dims, lstm_dims
        self.speaker_embedding_size = speaker_embedding_size
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_tacotron_create(C.byref(cfg), C.byref(self._handle)))
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena = None
        self._ws = None
        self._trim_ws = None
        self._device = None
        self._ready = False
        self._r = 1
        self.step = torch.zeros(1, dtype=torch.long)
        self.stop_threshold = torch.tensor(stop_threshold, dtype=torch.float32)
        self.training = True
        self.seed = 0

    # -- Base (base.py) ---------------------------------------------------------------------------
    @property
    def r(self):
        return self._r

    @r.setter
    def r(self, value):
        self._r = int(value)

    def get_step(self):
        return self.step.data.item()

    def load(self, path, device=None, optimizer=None):
        checkpoint = torch.load(str(path), map_location="cpu")
        state = checkpoint["model_state"] if "model_state" in checkpoint else checkpoint["model"]
        self.load_state_dict(state, strict=False)

    def load_state_dict(self, sd, strict: bool = True):
        self._state = {k: v.detach() for k, v in sd.items()}
        if "decoder.r" in self._state:
            self._r = int(self._state["decoder.r"])
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

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 Tacotron runs on CUDA only (no CPU fallback)")
        self._device = device
        self._ready = False
        return self

    def cuda(self):
        return self.to(_lib.require_cuda())

    # -- weights -----------------------------------------------------------------------------------
    def _gst_const_enc(self) -> torch.Tensor:
        """ReferenceEncoder(zeros) of tacotron.py:251 (global_style_token.py:56-72): the input is all
        zeros, so the result is a constant of the weights - folded here at load time (torch ops on
        the checkpoint tensors), like weight-norm folding in the GAN loaders."""
        sd = self._state
        out = torch.zeros(1, 1, 1, gst_hparams.n_mels)
        i = 0
        while f"gst.encoder.convs.{i}.weight" in sd:
            out = F.conv2d(out, sd[f"gst.encoder.convs.{i}.weight"].float(), sd[f"gst.encoder.convs.{i}.bias"].float(), 2, 1)
            p = f"gst.encoder.bns.{i}"
            out = F.batch_norm(out, sd[p + ".running_mean"].float(), sd[p + ".running_var"].float(), sd[p + ".weight"].float(),
                               sd[p + ".bias"].float(), False, 0.1, 1e-5)
            out = F.relu(out)
            i += 1
        x = out.transpose(1, 2).contiguous().view(1, -1)
        gi = F.linear(x, sd["gst.encoder.gru.weight_ih_l0"].float(), sd["gst.encoder.gru.bias_ih_l0"].float())
        gh = sd["gst.encoder.gru.bias_hh_l0"].float().unsqueeze(0)  # W_hh @ 0 + b_hh
        i_r, i_z, i_n = gi.chunk(3, 1)
        h_r, h_z, h_n = gh.chunk(3, 1)
        r = torch.sigmoid(h_r + i_r)
        z = torch.sigmoid(h_z + i_z)
        n = torch.tanh(i_n + h_n * r)
        return ((0.0 - n) * z + n).reshape(-1)

    def _upload(self):
        if self._state is None:
            raise _lib.MbError("Tacotron has no weights: call load_state_dict / load first")
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("tacotron", self._handle, self.weights_for_upload(), self._device)
        self._ready = True

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """the float tensors of the checkpoint without the GST reference encoder, which is folded into gst.const_enc"""
        tensors = {k: v for k, v in self._state.items()
                   if v.dtype.is_floating_point and not k.startswith("gst.encoder.") and k != "stop_threshold"}
        tensors["gst.const_enc"] = self._gst_const_enc()
        return tensors

    def packed_arena(self) -> torch.Tensor:
        if not self._ready:
            self._upload()
        return self._arena

    # -- generate ----------------------------------------------------------------------------------
    def generate(self, x, speaker_embedding, steps=2000, style_idx=0, min_stop_token=5, dropout_masks=None):
        self.eval()
        if not self._ready:
            self._upload()
        dev = self._device
        L = _lib.lib()
        chars = x.to(device=dev, dtype=torch.int32).contiguous()
        spk = speaker_embedding.to(device=dev, dtype=torch.float32).contiguous()
        B, Tc = chars.shape
        with torch.cuda.device(dev):
            max_chars = int(L.mb_tacotron_max_chars())
        if Tc > max_chars:
            raise ValueError(f"{Tc} characters exceed the limit of {max_chars} per utterance on this GPU "
                             "(the attention step keeps 4 * (5438 + 38 * chars) bytes in shared memory)")
        r = self._r
        nst = (steps + r - 1) // r
        M = nst * r
        mel = torch.empty(B * self.n_mels * M, dtype=torch.float32, device=dev)
        lin = torch.empty(B * self.n_mels * M, dtype=torch.float32, device=dev)
        attn = torch.empty(B * nst * Tc, dtype=torch.float32, device=dev)
        enc_p = dec_p = None
        if dropout_masks is not None:
            enc_m = dropout_masks[0].to(device=dev, dtype=torch.uint8).contiguous()
            dec_m = dropout_masks[1].to(device=dev, dtype=torch.uint8).contiguous()
            assert enc_m.numel() == 2 * B * Tc * self.encoder_dims and dec_m.numel() >= nst * 2 * B * 2 * self.decoder_dims
            enc_p, dec_p = C.c_void_p(enc_m.data_ptr()), C.c_void_p(dec_m.data_ptr())
        frames = C.c_int32(0)
        with torch.cuda.device(dev):
            need = int(L.mb_tacotron_workspace_bytes(self._handle, B, Tc, steps, r))
            _lib.workspace(need, dev, self)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(L.mb_tacotron_generate(self._handle, C.c_void_p(chars.data_ptr()), C.c_void_p(spk.data_ptr()), B, Tc,
                                              int(steps), r, int(style_idx), C.c_float(float(min_stop_token)), enc_p, dec_p,
                                              C.c_uint64(self.seed), C.c_void_p(mel.data_ptr()), C.c_void_p(lin.data_ptr()),
                                              C.c_void_p(attn.data_ptr()), C.byref(frames), C.c_void_p(self._ws.data_ptr()),
                                              self._ws.numel(), C.c_void_p(stream)))
        f = frames.value
        mel = mel[: B * self.n_mels * f].view(B, self.n_mels, f)
        lin = lin[: B * self.n_mels * f].view(B, self.n_mels, f)
        attn = attn[: B * (f // r) * Tc].view(B, f // r, Tc)
        return mel, lin, attn

    def _many_args(self, seqs, speaker_embeddings, steps, seeds, dropout_masks):
        """generate_many's argument checks -> (int32 rows, speaker embeddings [N, 256], frame caps, seeds)"""
        N = len(seqs)
        rows = [torch.as_tensor(s).reshape(-1).to(torch.int32) for s in seqs]
        L = _lib.lib()
        with torch.cuda.device(self._device or _lib.require_cuda()):
            max_chars = int(L.mb_tacotron_max_chars())
        for i, s in enumerate(rows):
            if s.numel() == 0:
                raise ValueError(f"text {i} is empty")
            if s.numel() > max_chars:
                raise ValueError(f"text {i} has {s.numel()} characters, over the limit of {max_chars} per utterance on this GPU")
        spk_all = torch.as_tensor(speaker_embeddings).to(dtype=torch.float32)
        if spk_all.dim() != 2 or spk_all.shape[0] != N or spk_all.shape[1] != self.speaker_embedding_size:
            raise ValueError(f"speaker_embeddings has shape {tuple(spk_all.shape)}, expected ({N}, {self.speaker_embedding_size})")
        caps = [int(steps)] * N if isinstance(steps, (int, np.integer)) else [int(v) for v in steps]
        if len(caps) != N:
            raise ValueError(f"{len(caps)} frame caps for {N} texts")
        if min(caps) < 1:
            raise ValueError("every frame cap must be at least 1")
        seeds = [self.seed + i for i in range(N)] if seeds is None else [int(v) for v in seeds]
        if len(seeds) != N:
            raise ValueError(f"{len(seeds)} seeds for {N} texts")
        r = self._r
        E, D2 = self.encoder_dims, 2 * self.decoder_dims
        if dropout_masks is not None:
            enc_l, dec_l = dropout_masks
            if len(enc_l) != N or len(dec_l) != N:
                raise ValueError(f"dropout_masks need {N} encoder and {N} decoder masks")
            for i in range(N):
                if tuple(enc_l[i].shape) != (2, rows[i].numel(), E):
                    raise ValueError(f"encoder mask {i} has shape {tuple(enc_l[i].shape)}, expected (2, {rows[i].numel()}, {E})")
                nst_i = -(-caps[i] // r)
                if enc_l[i].dim() != 3 or dec_l[i].dim() != 3 or dec_l[i].shape[0] < nst_i or tuple(dec_l[i].shape[1:]) != (2, D2):
                    raise ValueError(f"decoder mask {i} has shape {tuple(dec_l[i].shape)}, expected ({nst_i}, 2, {D2})")
        return rows, spk_all, caps, seeds

    def generate_many(self, seqs, speaker_embeddings, steps=2000, style_idx=0, min_stop_token=5, seeds=None,
                      dropout_masks=None, chunk_rows=None, trim_threshold=None):
        """Many texts, each computed as its own B = 1 ``generate`` -> list of N ``(mel [80, f_i], linear [80, f_i],
        attn [f_i / r, Tc_i])`` device tensors in input order.

        ``seqs``: N unpadded int sequences; ``speaker_embeddings`` [N, 256]; ``steps``: one frame cap or N of them.  Each
        utterance stops at its own stop rule or cap.  Utterances are sorted longest first and run in ragged batches of at
        most ``chunk_rows`` (default ``MANY_CHUNK_ROWS``) rows; a result is bitwise the same whatever the list around it.
        Dropout is drawn from ``seeds[i]`` (default ``self.seed + i``) or injected per utterance as
        ``dropout_masks = (enc, dec)`` with enc[i] [2, Tc_i, 256] and dec[i] [>= ceil(steps_i / r), 2, 256].
        ``trim_threshold`` (a float): each linear output is cut to its trailing-silence trim, the frames up to the last one
        whose largest channel is not below the threshold (synthesizer/inference.py:135-138), found on the device by one
        mb_tacotron_trim_frames launch per chunk; only the trimmed lengths come back to the host."""
        self.eval()
        N = len(seqs)
        if N == 0:
            return []
        rows, spk_all, caps, seeds = self._many_args(seqs, speaker_embeddings, steps, seeds, dropout_masks)
        L = _lib.lib()
        r = self._r
        E, D2 = self.encoder_dims, 2 * self.decoder_dims
        if dropout_masks is not None:
            enc_l, dec_l = dropout_masks
        if not self._ready:
            self._upload()
        dev = self._device
        out = [None] * N
        for chunk in many_plan([s.numel() for s in rows], chunk_rows or MANY_CHUNK_ROWS):
            B = len(chunk)
            Tc = max(rows[i].numel() for i in chunk)
            lens = [rows[i].numel() for i in chunk]
            ccaps = [caps[i] for i in chunk]
            nst = -(-max(ccaps) // r)
            M = nst * r
            chars = torch.zeros(B, Tc, dtype=torch.int32)
            for b, i in enumerate(chunk):
                chars[b, : lens[b]] = rows[i]
            chars = chars.to(dev)
            spk = spk_all[chunk].to(dev).contiguous()
            enc_p = dec_p = None
            if dropout_masks is not None:
                enc_m = torch.zeros(2, B, Tc, E, dtype=torch.uint8)
                dec_m = torch.zeros(nst, 2, B, D2, dtype=torch.uint8)
                for b, i in enumerate(chunk):
                    enc_m[:, b, : lens[b]] = enc_l[i].to(torch.uint8)
                    n_i = -(-caps[i] // r)
                    dec_m[:n_i, :, b] = dec_l[i][:n_i].to(torch.uint8)
                enc_m, dec_m = enc_m.to(dev), dec_m.to(dev)
                enc_p, dec_p = C.c_void_p(enc_m.data_ptr()), C.c_void_p(dec_m.data_ptr())
            mel = torch.empty(B * self.n_mels * M, dtype=torch.float32, device=dev)
            lin = torch.empty(B * self.n_mels * M, dtype=torch.float32, device=dev)
            attn = torch.empty(B * nst * Tc, dtype=torch.float32, device=dev)
            row_chars = (C.c_int32 * B)(*lens)
            row_steps = (C.c_int32 * B)(*ccaps)
            row_seeds = (C.c_uint64 * B)(*[seeds[i] & 0xFFFFFFFFFFFFFFFF for i in chunk])
            row_frames = (C.c_int32 * B)()
            frames = C.c_int32(0)
            with torch.cuda.device(dev):
                need = int(L.mb_tacotron_ragged_workspace_bytes(self._handle, B, Tc, max(ccaps), r))
                _lib.workspace(need, dev, self)
                stream = torch.cuda.current_stream(dev).cuda_stream
                _lib.check(L.mb_tacotron_generate_ragged(
                    self._handle, C.c_void_p(chars.data_ptr()), C.c_void_p(spk.data_ptr()), B, Tc, row_chars, row_steps,
                    row_seeds, r, int(style_idx), C.c_float(float(min_stop_token)), enc_p, dec_p, C.c_void_p(mel.data_ptr()),
                    C.c_void_p(lin.data_ptr()), C.c_void_p(attn.data_ptr()), C.byref(frames), row_frames,
                    C.c_void_p(self._ws.data_ptr()), self._ws.numel(), C.c_void_p(stream)))
            F_ = frames.value
            keep = list(row_frames)
            if trim_threshold is not None:
                keep = self._trim_frames(lin, B, F_, row_frames, float(trim_threshold))
            mel = mel[: B * self.n_mels * F_].view(B, self.n_mels, F_)
            lin = lin[: B * self.n_mels * F_].view(B, self.n_mels, F_)
            attn = attn[: B * (F_ // r) * Tc].view(B, F_ // r, Tc)
            for b, i in enumerate(chunk):
                f = row_frames[b]
                out[i] = (mel[b, :, :f].clone(), lin[b, :, :keep[b]].clone(), attn[b, : f // r, : lens[b]].clone())
        return out

    def _trim_frames(self, lin, B, F_, row_frames, threshold):
        """mb_tacotron_trim_frames over a chunk's postnet output [B, 80, F_] -> the B trimmed frame counts (host ints)"""
        L = _lib.lib()
        dev = self._device
        with torch.cuda.device(dev):
            kept = torch.empty(B, dtype=torch.int32, device=dev)
            ws = _lib.workspace(int(L.mb_tacotron_trim_workspace_bytes(B)), dev, self, "_trim_ws")
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(L.mb_tacotron_trim_frames(C.c_void_p(lin.data_ptr()), B, self.n_mels, F_, row_frames,
                                                 C.c_float(threshold), C.c_void_p(kept.data_ptr()), C.c_void_p(ws.data_ptr()),
                                                 ws.numel(), C.c_void_p(stream)))
            return kept.cpu().tolist()

    def generate_stream(self, seqs, speaker_embeddings, steps=2000, style_idx=0, min_stop_token=5, seeds=None,
                        dropout_masks=None, slots=MANY_CHUNK_ROWS):
        """Many texts through one decoder loop of ``slots`` rows (1..128): a text enters a free row as soon as one is free,
        and its result comes back as soon as its postnet has run -> iterator of ``(i, mel [80, f_i], linear [80, f_i],
        attn [f_i / r, Tc_i])`` device tensors in the order the texts finish, each bitwise what ``generate_many`` returns for
        text i.  Same arguments and checks as ``generate_many`` (checked before this returns).  Texts are admitted longest
        first, ties in input order, and encoded a batch of ``slots`` ahead on a stream of their own; the postnet runs on
        another stream over every row that finished since the previous postnet started.  Stopping early is allowed: the
        model stays usable.  ``self.stream_steps`` holds the decoder steps the loop has run."""
        self.eval()
        if not 1 <= int(slots) <= 128:
            raise ValueError(f"slots must be in [1, 128], got {slots}")
        N = len(seqs)
        if N == 0:
            return iter(())
        rows, spk_all, caps, seeds = self._many_args(seqs, speaker_embeddings, steps, seeds, dropout_masks)
        if not self._ready:
            self._upload()
        return self._stream(rows, spk_all, caps, seeds, int(style_idx), float(min_stop_token), dropout_masks, int(slots))

    def _stream(self, rows, spk_all, caps, seeds, style_idx, min_stop_token, dropout_masks, slots):
        L = _lib.lib()
        dev = self._device
        r, E = self._r, self.encoder_dims
        N = len(rows)
        lens = [s.numel() for s in rows]
        Tc, max_steps = max(lens), max(caps)
        sched = StreamSchedule(lens, slots)
        dec = None
        if dropout_masks is not None:  # each text's decoder masks for its steps, on the device while it may be admitted
            dec = [dropout_masks[1][i][: -(-caps[i] // r)].to(device=dev, dtype=torch.uint8).contiguous() for i in range(N)]
        with torch.cuda.device(dev):
            need = int(L.mb_tacotron_stream_workspace_bytes(self._handle, slots, Tc, max_steps, r))
            if need == 0:
                raise ValueError(f"no stream of {slots} rows for texts of {Tc} characters and {max_steps} frames")
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            cur = torch.cuda.current_stream(dev)
            post = torch.cuda.Stream(dev)
            post.wait_stream(cur)
            handle = C.c_void_p()
            _lib.check(L.mb_tacotron_stream_open(self._handle, slots, Tc, max_steps, r, style_idx, C.c_float(min_stop_token),
                                                 C.c_void_p(ws.data_ptr()), need, C.c_void_p(cur.cuda_stream), C.byref(handle)))
        keep = []          # device inputs of calls that may still be running (released at close)
        finished = []      # (text, frames) of rows run() reported and no postnet has taken yet
        flights = []       # postnets launched: (event, [(text, frames)], mel, linear, attn)
        slot_of = {}       # text -> slot while it decodes
        n_done = C.c_int32(0)
        ids = (C.c_int64 * slots)()
        frames = (C.c_int32 * slots)()
        steps_run = C.c_int64(0)
        self.stream_steps = 0
        try:
            while not sched.done() or finished or flights:
                with torch.cuda.device(dev):
                    for row0, batch in sched.to_encode():
                        n = len(batch)
                        chars = torch.zeros(n, Tc, dtype=torch.int32)
                        for b, i in enumerate(batch):
                            chars[b, : lens[i]] = rows[i]
                        chars = chars.to(dev)
                        spk = spk_all[batch].to(dev).contiguous()
                        enc_p = None
                        if dropout_masks is not None:
                            enc_m = torch.zeros(2, n, Tc, E, dtype=torch.uint8)
                            for b, i in enumerate(batch):
                                enc_m[:, b, : lens[i]] = dropout_masks[0][i].to(torch.uint8)
                            enc_m = enc_m.to(dev)
                            keep.append(enc_m)
                            enc_p = C.c_void_p(enc_m.data_ptr())
                        keep += [chars, spk]
                        _lib.check(L.mb_tacotron_stream_encode(
                            handle, row0, n, C.c_void_p(chars.data_ptr()), C.c_void_p(spk.data_ptr()),
                            (C.c_int32 * n)(*[lens[i] for i in batch]),
                            (C.c_uint64 * n)(*[seeds[i] & 0xFFFFFFFFFFFFFFFF for i in batch]), enc_p, C.c_void_p(cur.cuda_stream)))
                    adm = sched.admit()
                    if adm:
                        n = len(adm)
                        masks = None
                        if dec is not None:
                            masks = (C.c_void_p * n)(*[dec[i].data_ptr() for _, i, _ in adm])
                        _lib.check(L.mb_tacotron_stream_admit(
                            handle, n, (C.c_int32 * n)(*[s for s, _, _ in adm]), (C.c_int32 * n)(*[p for _, _, p in adm]),
                            (C.c_int64 * n)(*[i for _, i, _ in adm]), (C.c_int32 * n)(*[lens[i] for _, i, _ in adm]),
                            (C.c_int32 * n)(*[caps[i] for _, i, _ in adm]),
                            (C.c_uint64 * n)(*[seeds[i] & 0xFFFFFFFFFFFFFFFF for _, i, _ in adm]), masks,
                            C.c_void_p(cur.cuda_stream)))
                        for slot, i, _ in adm:
                            slot_of[i] = slot
                    if sched.busy():
                        _lib.check(L.mb_tacotron_stream_run(handle, C.byref(n_done), ids, frames, C.byref(steps_run)))
                        self.stream_steps = steps_run.value
                        for k in range(n_done.value):
                            finished.append((int(ids[k]), int(frames[k])))
                            sched.finish(slot_of.pop(int(ids[k])))
                    # one postnet over every row finished since the previous one started, once that one is done (or when
                    # nothing else is left to overlap with, or the finished rows would fill their pool)
                    idle = not flights or flights[-1][0].query()
                    if finished and (idle or len(finished) >= slots or sched.done()):
                        take, finished = finished[:slots], finished[slots:]
                        F = max(f for _, f in take)
                        n = len(take)
                        with torch.cuda.stream(post):
                            mel = torch.empty(n, self.n_mels, F, dtype=torch.float32, device=dev)
                            lin = torch.empty(n, self.n_mels, F, dtype=torch.float32, device=dev)
                            att = torch.empty(n, F // r, Tc, dtype=torch.float32, device=dev)
                        _lib.check(L.mb_tacotron_stream_harvest(handle, n, F, C.c_void_p(mel.data_ptr()),
                                                                C.c_void_p(lin.data_ptr()), C.c_void_p(att.data_ptr()),
                                                                C.c_void_p(post.cuda_stream)))
                        ev = torch.cuda.Event()
                        ev.record(post)
                        flights.append((ev, take, mel, lin, att))
                    ready = []
                    while flights and (flights[0][0].query() or (sched.done() and not finished)):
                        ev, take, mel, lin, att = flights.pop(0)
                        ev.synchronize()
                        cur.wait_event(ev)
                        for t in (mel, lin, att):
                            t.record_stream(cur)
                        for b, (i, f) in enumerate(take):
                            ready.append((i, mel[b, :, :f].clone(), lin[b, :, :f].clone(), att[b, : f // r, : lens[i]].clone()))
                yield from ready
        finally:
            with torch.cuda.device(dev):
                L.mb_tacotron_stream_close(handle)
                cur.wait_stream(post)

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_tacotron_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
