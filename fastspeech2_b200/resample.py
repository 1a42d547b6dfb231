"""Sample-rate conversion of synthesised speech on the GPU: scipy.signal.resample_poly(x, up, down) with its default Kaiser(5.0)
window and zero padding, computed by the polyphase FIR kernel behind fs2_resample / fs2_resample_window / fs2_resample_streams
(include/fs2b200.h states the formula and the order of the fp32 sums).  The taps are designed here in fp64 with numpy, as
scipy.signal.firwin designs them, so the runtime needs no scipy.

Mixed streams (Resampler.mixed, fs2_resample_streams_mixed): streams at different rates and encodings -- fp32, int16 PCM, or the
ITU-T G.711 mu-law / A-law byte of that PCM -- in one launch; a stream at the input rate that wants PCM or G.711 runs the identity
filter.  Generator.stream_pool converts every stream of a step this way.

Streaming: after m input samples of a stream have arrived, output j is ready iff floor((j * down + half_len) / up) < m, or the stream
has ended (Resampler.ready).  Generator.stream and Generator.stream_pool emit exactly the ready outputs on each chunk; an output's
arithmetic never depends on where a chunk boundary falls, so the concatenated chunks equal the offline call bit for bit.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers

import numpy as np
import torch

from . import _lib as L
from . import _streams

# output encodings of the mixed call, by name; a stream's chunk has the dtype of its encoding
ENCODINGS = {"f32": L.RESAMPLE_F32, "pcm16": L.RESAMPLE_PCM16, "ulaw": L.RESAMPLE_ULAW, "alaw": L.RESAMPLE_ALAW}
DTYPES = {L.RESAMPLE_F32: torch.float32, L.RESAMPLE_PCM16: torch.int16, L.RESAMPLE_ULAW: torch.uint8, L.RESAMPLE_ALAW: torch.uint8}
_UNIT_TAP = np.ones((1, 1), dtype=np.float32)       # the identity filter: up = down = K = 1


def _rate(v, name):
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not float(v).is_integer() or v <= 0:
        raise ValueError(f"{name} must be a positive integer rate in Hz, got {v!r}")
    return int(v)


def design_taps(up: int, down: int) -> np.ndarray:
    """resample_poly's filter in fp64: firwin(2 half_len + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up, half_len =
    10 max(up, down).  Symmetric Kaiser window, windowed sinc, unit DC gain, then the gain `up` of the zero-stuffing."""
    mx = max(up, down)
    half_len = 10 * mx
    n = 2 * half_len + 1
    m = np.arange(n, dtype=np.float64) - 0.5 * (n - 1)
    cutoff = 1.0 / mx
    h = cutoff * np.sinc(cutoff * m) * np.kaiser(n, 5.0)
    return h / h.sum() * up


def polyphase(h: np.ndarray, up: int) -> np.ndarray:
    """[up][K] fp32, row p = h[p], h[p + up], h[p + 2 up], ... zero-filled past the filter; K = ceil(len(h) / up)."""
    K = -(-len(h) // up)
    pad = np.zeros(K * up, dtype=np.float64)
    pad[:len(h)] = h
    return np.ascontiguousarray(pad.reshape(K, up).T.astype(np.float32))


class Resampler:
    """Converts waveforms from fs_in to fs_out Hz (up / down = fs_out / fs_in reduced).  fs_out == fs_in is the identity: the input is
    returned unchanged, with no launch.  Refuses non-positive or non-integer rates and max(up, down) > 2048 with ValueError.

    CUDA streams: every call (__call__, window, streams, mixed) enqueues all of its device work on the stream current at that call.
    The waveforms, lengths and records the caller passes in and the outputs it gets back follow torch's usual rule: the caller orders
    them across streams.  The taps, uploaded to a device by the first call there, are ready on whatever stream a later call uses."""

    def __init__(self, fs_in, fs_out):
        self.fs_in, self.fs_out = _rate(fs_in, "fs_in"), _rate(fs_out, "fs_out")
        g = math.gcd(self.fs_in, self.fs_out)
        self.up, self.down = self.fs_out // g, self.fs_in // g
        if max(self.up, self.down) > L.RESAMPLE_MAX_FACTOR:
            raise ValueError(f"{self.fs_in} -> {self.fs_out} Hz needs up/down = {self.up}/{self.down}; "
                             f"max(up, down) must be <= {L.RESAMPLE_MAX_FACTOR}")
        self.identity = self.up == self.down
        self.half_len = 10 * max(self.up, self.down)
        self.K = -(-(2 * self.half_len + 1) // self.up)
        self.taps = None if self.identity else polyphase(design_taps(self.up, self.down), self.up)
        self._dev_taps = {}

    def n_out(self, n: int) -> int:
        """Outputs of n input samples: ceil(n * up / down)."""
        return -(-n * self.up // self.down)

    @property
    def history(self) -> int:
        """Input samples before the first not-yet-emitted output's support that a window may still need: K - 1."""
        return 0 if self.identity else self.K - 1

    def ready(self, m: int, n: int | None, ended: bool) -> int:
        """Outputs ready once m of a stream's n input samples have arrived: j is ready iff floor((j down + half_len) / up) < m, or
        the stream has ended (then all n_out(n)).  n None: a stream whose length is not known yet, which has not ended; its ready
        outputs are not capped at n_out(n)."""
        if ended:
            return self.n_out(n)
        r = m if self.identity else max(0, -(-(m * self.up - self.half_len) // self.down))
        return r if n is None else min(self.n_out(n), r)

    def device_taps(self, device):
        """The [up][K] taps on `device` (the identity: the one-tap table of 1.0 that the mixed call runs), uploaded once."""
        device = torch.device(device)
        t = self._dev_taps.get(device)
        if t is None:
            tab = torch.from_numpy(_UNIT_TAP if self.identity else self.taps).to(device)
            t = self._dev_taps[device] = (tab, _streams.made(device))     # the upload is ordered on the current stream only
        t[1].enter()
        return t[0]

    def _filter(self, device):
        return dict(up=self.up, down=self.down, K=1 if self.identity else self.K, taps=self.device_taps(device).data_ptr())

    @torch.no_grad()
    def __call__(self, wav, lengths=None, pcm16=False, scale=32768.0):
        """wav: fp32 [B, N] or [B, 1, N] on a CUDA device, any strides.  lengths (optional): integer [B] of input samples per row, on
        any device; row b is then resampled over its first lengths[b] samples exactly as alone, and its outputs at or past
        ceil(lengths[b] * up / down) are zeros (a CPU tensor is range-checked to [0, N], device values are clamped).  Returns fp32, or
        int16 = trunc(y * scale) clamped to the int16 range when pcm16, of shape [B, ceil(N up / down)] or [B, 1, ...], on the
        current stream.  The identity ratio returns wav itself (pcm16: its int16 conversion), lengths unused."""
        if not isinstance(wav, torch.Tensor) or wav.dim() not in (2, 3) or (wav.dim() == 3 and wav.shape[1] != 1):
            raise ValueError("wav must be a [B, N] or [B, 1, N] tensor")
        if wav.device.type != "cuda":
            raise L.Fs2Error("Resampler runs on CUDA tensors; there is no CPU path")
        x = wav.reshape(wav.shape[0], wav.shape[-1]) if wav.dim() == 3 else wav
        B, N = x.shape
        if B < 1 or N < 1:
            raise ValueError("wav has no samples")
        if self.identity and not pcm16:
            return wav
        if x.dtype != torch.float32 or x.stride(1) != 1:
            x = x.to(torch.float32).contiguous()
        lens = None
        if lengths is not None:
            lengths = torch.as_tensor(lengths)
            if lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool or lengths.shape != (B,):
                raise ValueError(f"lengths must be an integer tensor of shape [{B}]")
            if lengths.device.type == "cpu" and not bool(((lengths >= 0) & (lengths <= N)).all()):
                raise ValueError(f"lengths must lie in [0, {N}]")
        dev = x.device
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            if self.identity:
                from . import ops
                y = ops.wav_to_int16(x, lengths, scale)
            else:
                if lengths is not None:
                    lens = lengths.to(device=dev, dtype=torch.int32).contiguous()
                n_out = self.n_out(N)
                y = torch.empty(B, n_out, dtype=torch.int16 if pcm16 else torch.float32, device=dev)
                a = L.ResampleArgs(B=B, x=x.data_ptr(), x_batch_stride=x.stride(0), N=N, lens=L.ptr(lens), lens_scale=1, y=y.data_ptr(),
                                   y_batch_stride=n_out, pcm16=int(bool(pcm16)), scale=float(scale), **self._filter(dev))
                L.check(L.lib().fs2_resample(C.byref(a), stream), "fs2_resample")
        return y.unsqueeze(1) if wav.dim() == 3 else y

    def window(self, prev, cur, i1, N, j0, j1, lens=None, lens_scale=1, pcm16=False, scale=32768.0):
        """Outputs [j0, j1) of every row into a new [B, j1 - j0] tensor (fs2_resample_window), from input samples [i1 - prev_len, i1)
        in prev ([B, prev_len] or None) and [i1, i1 + cur_len) in cur ([B, cur_len]); rows of N samples, bounded by the device lens
        (int32 [B], times lens_scale) when given.  Raises Fs2Error when an input the outputs need is missing."""
        B, n1 = cur.shape
        n0 = 0 if prev is None else prev.shape[1]
        dev = cur.device
        y = torch.empty(B, j1 - j0, dtype=torch.int16 if pcm16 else torch.float32, device=dev)
        a = L.ResampleWindowArgs(B=B, x0=L.ptr(prev), x0_batch_stride=0 if prev is None else prev.stride(0), x1=cur.data_ptr(),
                                 x1_batch_stride=cur.stride(0), i0=i1 - n0, i1=i1, i2=i1 + n1, N=N, lens=L.ptr(lens),
                                 lens_scale=lens_scale, j0=j0, j1=j1, y=y.data_ptr(), y_batch_stride=j1 - j0, pcm16=int(bool(pcm16)),
                                 scale=float(scale), **self._filter(dev))
        L.check(L.lib().fs2_resample_window(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "fs2_resample_window")
        return y

    def streams(self, records, max_out, device, pcm16=False, scale=32768.0):
        """One fs2_resample_streams launch: records[b] = (x0 pointer, x1 pointer, i0, i1, i2, n, j0, j1) of stream b, uploaded from a
        fresh pinned block with one non_blocking copy (no host sync).  Returns the [B, max_out] output; stream b's outputs are its
        first j1 - j0 columns."""
        B = len(records)
        dev = torch.device(device)
        host = torch.empty(8 * B, dtype=torch.int64, pin_memory=True)
        host.numpy()[:] = np.asarray(records, dtype=np.int64).reshape(-1)
        table = host.to(dev, non_blocking=True)
        y = torch.empty(B, max_out, dtype=torch.int16 if pcm16 else torch.float32, device=dev)
        a = L.ResampleStreamsArgs(B=B, table=table.data_ptr(), max_out=max_out, y=y.data_ptr(), y_batch_stride=max_out,
                                  pcm16=int(bool(pcm16)), scale=float(scale), **self._filter(dev))
        L.check(L.lib().fs2_resample_streams(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "fs2_resample_streams")
        return y

    @staticmethod
    def mixed_table(records, max_out):
        """The host side of Resampler.mixed, without device work: (filters, table, offsets, nbytes).  filters: the distinct ratios'
        Resamplers in order of first use (at most 8, else ValueError); table: int64 [B, 10], row b the fs2_resample_mixed_stream_t of
        stream b (its filter index and encoding packed as two int32 in column 8); offsets: stream b's byte offset in the output, each a
        multiple of 16, the streams back to back; nbytes: the output's size."""
        filters, index = [], {}
        table = np.zeros((len(records), 10), dtype=np.int64)
        offsets, off = [], 0
        for b, rec in enumerate(records):
            rs, enc = rec[8], rec[9]
            if enc not in DTYPES:
                raise ValueError(f"unknown encoding {enc!r}")
            k = index.get((rs.up, rs.down))
            if k is None:
                k = index[(rs.up, rs.down)] = len(filters)
                filters.append(rs)
            table[b, :8] = rec[:8]
            table[b, 8] = k | (enc << 32)
            table[b, 9] = off
            offsets.append(off)
            width = min(max(rec[7] - rec[6], 0), max_out) * DTYPES[enc].itemsize
            off += -(-width // 16) * 16
        if len(filters) > L.RESAMPLE_MAX_FILTERS:
            raise ValueError(f"{len(filters)} filters in one call; at most {L.RESAMPLE_MAX_FILTERS}")
        return filters, table, offsets, off

    @staticmethod
    def mixed(records, max_out, device, scale=32768.0):
        """One fs2_resample_streams_mixed launch on the current stream: records[b] = (x0, x1, i0, i1, i2, n, j0, j1, resampler,
        encoding) -- the fields of Resampler.streams' records, then stream b's Resampler (the identity included) and its encoding (an
        L.RESAMPLE_* code).  The records are uploaded from a fresh pinned block with one non_blocking copy (no host sync).  Returns
        (y, views): one uint8 buffer holding every stream's outputs, and stream b's min(j1 - j0, max_out) outputs as a view of it
        typed by its encoding (fp32, int16 or uint8).  max_out == 0: no launch, empty views."""
        dev = torch.device(device)
        filters, table, offsets, nbytes = Resampler.mixed_table(records, max_out)
        y = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
        views = []
        for rec, off in zip(records, offsets):
            dt = DTYPES[rec[9]]
            views.append(y[off:off + min(max(rec[7] - rec[6], 0), max_out) * dt.itemsize].view(dt))
        if max_out > 0 and records:
            host = torch.empty(table.size, dtype=torch.int64, pin_memory=True)
            host.numpy()[:] = table.reshape(-1)
            dtable = host.to(dev, non_blocking=True)
            a = L.ResampleMixedArgs(B=len(records), n_filters=len(filters), table=dtable.data_ptr(), max_out=max_out, y=y.data_ptr(),
                                    scale=float(scale))
            for i, rs in enumerate(filters):
                a.filters[i] = L.ResampleFilter(**rs._filter(dev))
            L.check(L.lib().fs2_resample_streams_mixed(C.byref(a), torch.cuda.current_stream(dev).cuda_stream),
                    "fs2_resample_streams_mixed")
        return y, views
