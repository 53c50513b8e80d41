"""Audio at the client's sample rate and encoding: a streaming, per-row GPU resampler (q3_resample_*, csrc/resample.cu).

The conversion is scipy.signal.resample_poly's: for a rate pair sr_in -> sr_out, up/down = sr_out/sr_in reduced, the
taps h = firwin(2*hl + 1, 1/max(up, down), window=("kaiser", 5.0)) * up with hl = 10*max(up, down) are designed here in
fp64 and uploaded as fp32, and a clip x[0..n) becomes ceil(n*up/down) samples
    y[j] = sum_m x[m] * h[hl + j*down - m*up]      over 0 <= m < n and 0 <= hl + j*down - m*up <= 2*hl,
summed in fp32 on the GPU.  Equal rates are a copy (resample_poly with up = down = 1).  The encoding is applied to y in
the same kernel: "f32" as is, "s16" clamp(rint(y * 32768), -32768, 32767) with round-half-even, "ulaw" the G.711 mu-law
of that int16 as audioop.lin2ulaw(..., 2) computes it.

Streaming: each row keeps its filter, encoding, input count and last inputs on the device.  Output j of a row is
emitted as soon as input floor((hl + j*down) / up) has arrived, so after n inputs a row has emitted emitted(n) samples;
an end emits the rest, as if the clip were followed by zeros.  A clip pushed in pieces of any sizes and ended equals
oneshot() of the whole clip bit for bit, and one launch serves every row of a push.

Speaking rate: TimeStretch, a streaming per-row WSOLA time-stretch at 24 kHz (q3_stretch_*, csrc/stretch.cu, DESIGN
§4.7), with the same streaming contract; the batcher runs it before the resampler.
"""
import ctypes as C
from math import gcd
from typing import Dict, Iterable, List, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .codec_encoder import check_chunks, check_rows
from .config import ENCODINGS, SUPPORTED_RATES, AudioFormat

CODEC_RATE = 24000                 # the codec's sample rate: decoder output and encoder input
ROW_BYTES = 528                    # Q3_RESAMPLE_ROW_BYTES: one row's saved state
_ENC_CODE = {e: i for i, e in enumerate(ENCODINGS)}           # Q3_RESAMPLE_F32 / S16 / ULAW
_ENC_DTYPE = {"f32": torch.float32, "s16": torch.int16, "ulaw": torch.uint8}
_NP_DTYPE = {"f32": np.float32, "s16": np.int16, "ulaw": np.uint8}
_WIDTH = {"f32": 4, "s16": 2, "ulaw": 1}


def ratio(sr_in: int, sr_out: int) -> Tuple[int, int]:
    """(up, down): sr_out / sr_in in lowest terms.  ValueError for a rate outside SUPPORTED_RATES."""
    for sr in (sr_in, sr_out):
        if isinstance(sr, bool) or not isinstance(sr, (int, np.integer)) or int(sr) not in SUPPORTED_RATES:
            raise ValueError(f"sample rate {sr!r} is not supported; supported rates: {SUPPORTED_RATES}")
    g = gcd(int(sr_in), int(sr_out))
    return int(sr_out) // g, int(sr_in) // g


def half_len(up: int, down: int) -> int:
    """hl: the filter has 2*hl + 1 taps (0 for equal rates)."""
    return 0 if up == down else 10 * max(up, down)


def design(up: int, down: int) -> np.ndarray:
    """The fp64 taps resample_poly designs for up/down ([1.0] for equal rates)."""
    if up == down:
        return np.ones(1)
    from scipy.signal import firwin
    hl = half_len(up, down)
    return firwin(2 * hl + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up


def emitted(n: int, up: int, down: int) -> int:
    """Outputs a row has emitted after n inputs without an end: max(0, floor((n*up - 1 - hl) / down) + 1)."""
    return max(0, (n * up - 1 - half_len(up, down)) // down + 1)


def total(n: int, up: int, down: int) -> int:
    """Outputs of a whole clip of n inputs: ceil(n*up / down)."""
    return -(-n * up // down)


def out_bound(max_in: int, up: int, down: int) -> int:
    """The most outputs one push of max_in inputs plus its end can emit (the native add-filter check)."""
    return -(-max_in * up // down) + -(-half_len(up, down) // down) + 1


def check_format(fmt) -> AudioFormat:
    if not isinstance(fmt, AudioFormat):
        raise ValueError(f"an audio format must be an AudioFormat, got {type(fmt).__name__}")
    return fmt


class Resampler:
    """`rows` streaming resampler rows on `device`; a push gives each row at most `max_in` samples per launch (longer
    pushes take several launches).  reset(rows, in_rate, fmt) starts new clips; push({row: samples}, end=rows) returns
    {row: numpy array of the row's new output} in the row's encoding (float32, int16 or uint8); push_device keeps them
    on the device; save(rows) / load(rows, state) move rows' state; oneshot(x, in_rate, fmt) converts a whole clip."""

    def __init__(self, device, rows: int, max_in: int):
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("Resampler needs a CUDA device (no CPU fallback)")
        self.rows, self.max_in = int(rows), int(max_in)
        # capacity for the widest supported pair, so any pair can be added later
        self.max_out = max(out_bound(self.max_in, *ratio(a, b)) for a in SUPPORTED_RATES for b in SUPPORTED_RATES)
        h = C.c_void_p()
        _lib.check(self.lib.q3_resample_open(self.rows, self.max_in, self.max_out, self.device.index or 0, C.byref(h)))
        self.h = h
        self._filters: Dict[Tuple[int, int], int] = {}
        self._enc: List[Optional[str]] = [None] * self.rows
        self._out = torch.empty(self.rows, 4 * self.max_out, dtype=torch.uint8, device=self.device)

    def close(self):
        if getattr(self, "h", None):
            self.lib.q3_resample_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        if not self.h:
            raise RuntimeError("resampler is closed")
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _filter(self, up: int, down: int) -> int:
        fid = self._filters.get((up, down))
        if fid is None:
            taps = torch.from_numpy(design(up, down)).to(self.device, torch.float32)
            out = C.c_int32()
            _lib.check(self.lib.q3_resample_add_filter(self.h, up, down, taps.data_ptr(), taps.numel(), C.byref(out)))
            fid = self._filters[(up, down)] = out.value
        return fid

    def reset(self, rows, in_rate: int, fmt: AudioFormat):
        """Start new clips in `rows` converting in_rate -> fmt.sample_rate into fmt.encoding."""
        rows = check_rows(rows, self.rows)
        fmt = check_format(fmt)
        fid = self._filter(*ratio(in_rate, fmt.sample_rate))
        n = len(rows)
        if n == 0:
            return
        i32n = C.c_int32 * n
        _lib.check(self.lib.q3_resample_reset_rows(self.h, n, i32n(*rows), i32n(*[fid] * n),
                                                   i32n(*[_ENC_CODE[fmt.encoding]] * n)))
        for r in rows:
            self._enc[r] = fmt.encoding

    def _check_ready(self, rows):
        for r in rows:
            if self._enc[r] is None:
                raise ValueError(f"row {r} was never reset")

    def _run(self, x: Optional[torch.Tensor], cnt: List[int], end: List[int], host: bool, listed=()) -> Dict[int, object]:
        """Row r takes x[r, :cnt[r]] and the rows in `end` end their clips, in launches of at most max_in samples per
        row; a row ends in the launch that takes its last sample.  Each launch's outputs reach the host in one copy
        (host=True) or stay on the device.  Returns {row: its new output} for rows with samples or an end and the rows
        `listed`."""
        if x is not None and (x.dim() != 2 or x.shape[0] != self.rows or x.dtype != torch.float32
                              or x.device != self.device or x.stride(1) != 1 or max(cnt) > x.shape[1]):
            raise ValueError(f"expected fp32 samples of shape ({self.rows}, L >= counts) on {self.device}")
        if x is None and any(cnt):
            raise ValueError("counts without samples")
        touched = sorted(set(end) | set(listed) | {r for r in range(self.rows) if cnt[r]})
        self._check_ready(touched)
        st = self._stream()
        parts: Dict[int, list] = {r: [] for r in touched}
        for s0 in range(0, max(max(cnt), 1), self.max_in):
            k = [min(max(c - s0, 0), self.max_in) for c in cnt]
            e = [int(r in end and (s0 == 0 if cnt[r] == 0 else s0 < cnt[r] <= s0 + self.max_in)) for r in range(self.rows)]
            nout = (C.c_int32 * self.rows)()
            ptr = x.data_ptr() + 4 * s0 if x is not None and any(k) else None
            _lib.check(self.lib.q3_resample_step_rows(self.h, ptr, x.stride(0) if x is not None else 0,
                                                      (C.c_int32 * self.rows)(*k), (C.c_int32 * self.rows)(*e),
                                                      self._out.data_ptr(), nout, st))
            nb = {r: nout[r] * _WIDTH[self._enc[r]] for r in touched}
            if host:
                top = max(nb.values(), default=0)
                buf = self._out[:, :top].cpu().numpy() if top else None
                for r in touched:
                    parts[r].append(buf[r, :nb[r]].view(_NP_DTYPE[self._enc[r]]) if nb[r] else None)
            else:
                for r in touched:
                    parts[r].append(self._out[r, :nb[r]].clone().view(_ENC_DTYPE[self._enc[r]]) if nb[r] else None)
        out = {}
        for r in touched:
            v = [p for p in parts[r] if p is not None]
            if host:
                out[r] = np.concatenate(v) if v else np.zeros(0, _NP_DTYPE[self._enc[r]])
            else:
                out[r] = torch.cat(v) if v else torch.zeros(0, dtype=_ENC_DTYPE[self._enc[r]], device=self.device)
        return out

    def push_rows(self, x: Optional[torch.Tensor], counts: Dict[int, int], end: Iterable[int] = (), host: bool = True):
        """Row r takes x[r, :counts[r]] of x, fp32 (rows, L) on the device with contiguous rows (the layout the codec
        stream returns), and the rows in `end` end their clips: one launch per max_in samples.  Returns {row: its new
        output} (numpy arrays when `host`, else device tensors) for every row with samples or an end."""
        cnt = [0] * self.rows
        for r, k in counts.items():
            if int(k) < 0:
                raise ValueError(f"row {r}: negative count {k}")
            cnt[check_rows(r, self.rows)[0]] = int(k)
        return self._run(x, cnt, check_rows(end, self.rows), host, listed=[int(r) for r in counts])

    def _pack(self, chunks: Dict, end) -> Tuple[Optional[torch.Tensor], Dict[int, int], List[int]]:
        chunks = check_chunks(chunks, self.rows)
        end = check_rows(end, self.rows)
        L = max([t.numel() for t in chunks.values()], default=0)
        if L == 0:
            return None, {r: 0 for r in chunks}, end
        on_dev = any(t.device.type == "cuda" for t in chunks.values())
        x = torch.zeros(self.rows, L, dtype=torch.float32, device=self.device if on_dev else "cpu")
        for r, t in chunks.items():
            x[r, : t.numel()] = t.to(x.device)
        return x.to(self.device), {r: t.numel() for r, t in chunks.items()}, end

    def push(self, chunks: Dict, end: Iterable[int] = ()) -> Dict[int, np.ndarray]:
        """chunks {row: 1-D float samples at the row's input rate} (numpy or torch, any length); the rows in `end` end
        their clips after their samples.  Returns {row: numpy array of its new output} for every row of chunks or
        end, float32, int16 or uint8 by the row's encoding.  One device-to-host copy per launch."""
        x, counts, end = self._pack(chunks, end)
        out = self.push_rows(x, counts, end, host=True)
        return {r: out[r] for r in sorted(set(chunks) | set(end))}

    def push_device(self, chunks: Dict, end: Iterable[int] = ()) -> Dict[int, torch.Tensor]:
        """push() with the outputs left on the device (for the encoder stream)."""
        x, counts, end = self._pack(chunks, end)
        out = self.push_rows(x, counts, end, host=False)
        return {r: out[r] for r in sorted(set(chunks) | set(end))}

    def save(self, rows) -> torch.Tensor:
        """The rows' state (filter, encoding, inputs so far, history): a uint8 (len(rows), ROW_BYTES) device tensor."""
        rows = check_rows(rows, self.rows)
        self._check_ready(rows)
        state = torch.empty(len(rows), ROW_BYTES, dtype=torch.uint8, device=self.device)
        n = len(rows)
        if n:
            _lib.check(self.lib.q3_resample_save_rows(self.h, n, (C.c_int32 * n)(*rows), state.data_ptr(), self._stream()))
        return state

    def load(self, rows, state: torch.Tensor):
        """Rows `rows` continue the states save() returned (of this resampler), in order."""
        rows = check_rows(rows, self.rows)
        if not isinstance(state, torch.Tensor) or state.dtype != torch.uint8 or tuple(state.shape) != (len(rows), ROW_BYTES) \
                or state.device != self.device:
            raise ValueError(f"expected a saved state of shape ({len(rows)}, {ROW_BYTES}) on {self.device}")
        n = len(rows)
        if n == 0:
            return
        state = state.contiguous()
        _lib.check(self.lib.q3_resample_load_rows(self.h, n, (C.c_int32 * n)(*rows), state.data_ptr(), self._stream()))
        inv = {v: k for k, v in _ENC_CODE.items()}
        codes = state[:, 4:8].cpu().numpy().view(np.int32)[:, 0]   # the header's encoding (already read back natively)
        for r, c in zip(rows, codes):
            self._enc[r] = inv[int(c)]

    def oneshot(self, x, in_rate: int, fmt: AudioFormat) -> np.ndarray:
        """The whole clip x (1-D float samples at in_rate) converted at once: the reference of the streamed result."""
        t = check_chunks({0: x}, 1)[0]
        one = Resampler(self.device, 1, max(t.numel(), 1))
        try:
            one.reset([0], in_rate, fmt)
            return one.push({0: t}, end=[0])[0]
        finally:
            one.close()


class TimeStretch:
    """`rows` streaming WSOLA time-stretch rows at the codec's 24 kHz on `device` (q3_stretch_*, csrc/stretch.cu, DESIGN
    §4.7): the speaking rate of float32 audio changes, its pitch does not.  Frames of N = 960 samples, synthesis hop
    480, search tolerance 240, analysis hop Ha = hop(speed) in [240, 960], window sin^2(pi*n/960).  A clip of n samples
    becomes total(n, Ha) samples; after n samples without an end a row has emitted emitted(n, Ha).  A push gives each
    row at most `max_in` samples per launch (longer pushes take several launches).  reset(rows, speed) starts new clips;
    push({row: samples}, end=rows) returns {row: float32 numpy array of the row's new output}; push_device keeps them on
    the device; save(rows) / load(rows, state) move rows' state; oneshot(x, speed) stretches a whole clip.  A clip pushed
    in pieces of any sizes and ended equals oneshot() of the whole clip bit for bit."""

    N, HS, DELTA = 960, 480, 240
    HIST = 2048                       # Q3_STRETCH_HIST: inputs a row keeps
    ROW_BYTES = 10144                 # Q3_STRETCH_ROW_BYTES: one row's saved state
    MAX_IN = 32768                    # the largest max_in the native stretcher takes

    @staticmethod
    def hop(speed) -> int:
        """The analysis hop of `speed`: floor(speed*480 + 0.5); the effective speed is hop/480.  ValueError outside
        [0.5, 2.0] (AudioFormat's check)."""
        return int(np.floor(AudioFormat(CODEC_RATE, speed=speed).speed * 480 + 0.5))

    @staticmethod
    def emitted(n: int, ha: int) -> int:
        """Outputs a row has emitted after n inputs without an end: 480*(floor((n - 1200)/Ha) + 1), 0 for n < 1200."""
        return 0 if n < 1200 else 480 * ((n - 1200) // ha + 1)

    @staticmethod
    def total(n: int, ha: int) -> int:
        """Outputs of a whole clip of n inputs: ceil(n*480 / Ha)."""
        return -(-n * 480 // ha)

    @staticmethod
    def out_bound(max_in: int, ha: int = 240) -> int:
        """The most outputs one push of max_in inputs plus its end can emit: ceil((max_in + 1199)*480 / Ha) (the
        slowest speed by default)."""
        return -(-(max_in + 1199) * 480 // ha)

    @staticmethod
    def window() -> np.ndarray:
        """w[n] = sin^2(pi*n/960), n in [0, 960), in fp64 (uploaded as fp32)."""
        return np.sin(np.pi * np.arange(960) / 960) ** 2

    def __init__(self, device, rows: int, max_in: int):
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("TimeStretch needs a CUDA device (no CPU fallback)")
        self.rows, self.max_in = int(rows), int(max_in)
        if not 1 <= self.max_in <= self.MAX_IN:
            raise ValueError(f"max_in {max_in} outside [1, {self.MAX_IN}]")
        self.max_out = self.out_bound(self.max_in)
        h = C.c_void_p()
        _lib.check(self.lib.q3_stretch_open(self.rows, self.max_in, self.max_out, self.device.index or 0, C.byref(h)))
        self.h = h
        w = torch.from_numpy(self.window()).to(self.device, torch.float32)
        _lib.check(self.lib.q3_stretch_set_window(self.h, w.data_ptr()))
        self._ha: List[Optional[int]] = [None] * self.rows
        self._out = torch.empty(self.rows, self.max_out, dtype=torch.float32, device=self.device)

    def close(self):
        if getattr(self, "h", None):
            self.lib.q3_stretch_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        if not self.h:
            raise RuntimeError("time-stretch is closed")
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def reset(self, rows, speed):
        """Start new clips in `rows` at `speed` (analysis hop hop(speed))."""
        rows = check_rows(rows, self.rows)
        ha = self.hop(speed)
        n = len(rows)
        if n == 0:
            return
        i32n = C.c_int32 * n
        _lib.check(self.lib.q3_stretch_reset_rows(self.h, n, i32n(*rows), i32n(*[ha] * n)))
        for r in rows:
            self._ha[r] = ha

    def _check_ready(self, rows):
        for r in rows:
            if self._ha[r] is None:
                raise ValueError(f"row {r} was never reset")

    def _run(self, x: Optional[torch.Tensor], cnt: List[int], end: List[int], host: bool, listed=()):
        """Resampler._run for the stretch: launches of at most max_in samples per row, a row ends in the launch that
        takes its last sample; returns {row: float32 output} for rows with samples or an end and the rows `listed`."""
        if x is not None and (x.dim() != 2 or x.shape[0] != self.rows or x.dtype != torch.float32
                              or x.device != self.device or x.stride(1) != 1 or max(cnt) > x.shape[1]):
            raise ValueError(f"expected fp32 samples of shape ({self.rows}, L >= counts) on {self.device}")
        if x is None and any(cnt):
            raise ValueError("counts without samples")
        touched = sorted(set(end) | set(listed) | {r for r in range(self.rows) if cnt[r]})
        self._check_ready(touched)
        st = self._stream()
        parts: Dict[int, list] = {r: [] for r in touched}
        for s0 in range(0, max(max(cnt), 1), self.max_in):
            k = [min(max(c - s0, 0), self.max_in) for c in cnt]
            e = [int(r in end and (s0 == 0 if cnt[r] == 0 else s0 < cnt[r] <= s0 + self.max_in)) for r in range(self.rows)]
            nout = (C.c_int32 * self.rows)()
            ptr = x.data_ptr() + 4 * s0 if x is not None and any(k) else None
            _lib.check(self.lib.q3_stretch_step_rows(self.h, ptr, x.stride(0) if x is not None else 0,
                                                     (C.c_int32 * self.rows)(*k), (C.c_int32 * self.rows)(*e),
                                                     self._out.data_ptr(), nout, st))
            nb = {r: nout[r] for r in touched}
            if host:
                top = max(nb.values(), default=0)
                buf = self._out[:, :top].cpu().numpy() if top else None
                for r in touched:
                    parts[r].append(buf[r, :nb[r]].copy() if nb[r] else None)
            else:
                for r in touched:
                    parts[r].append(self._out[r, :nb[r]].clone() if nb[r] else None)
        out = {}
        for r in touched:
            v = [p for p in parts[r] if p is not None]
            if host:
                out[r] = np.concatenate(v) if v else np.zeros(0, np.float32)
            else:
                out[r] = torch.cat(v) if v else torch.zeros(0, dtype=torch.float32, device=self.device)
        return out

    def push_rows(self, x: Optional[torch.Tensor], counts: Dict[int, int], end: Iterable[int] = (), host: bool = True):
        """Row r takes x[r, :counts[r]] of x, fp32 (rows, L) on the device with contiguous rows, and the rows in `end`
        end their clips: one launch per max_in samples.  Returns {row: its new float32 output} (numpy arrays when
        `host`, else device tensors) for every row with samples or an end and every row of `counts`."""
        cnt = [0] * self.rows
        for r, k in counts.items():
            if int(k) < 0:
                raise ValueError(f"row {r}: negative count {k}")
            cnt[check_rows(r, self.rows)[0]] = int(k)
        return self._run(x, cnt, check_rows(end, self.rows), host, listed=[int(r) for r in counts])

    _pack = Resampler._pack

    def push(self, chunks: Dict, end: Iterable[int] = ()) -> Dict[int, np.ndarray]:
        """chunks {row: 1-D float samples at 24 kHz} (numpy or torch, any length); the rows in `end` end their clips
        after their samples.  Returns {row: float32 numpy array of its new output} for every row of chunks or end."""
        x, counts, end = self._pack(chunks, end)
        out = self.push_rows(x, counts, end, host=True)
        return {r: out[r] for r in sorted(set(chunks) | set(end))}

    def push_device(self, chunks: Dict, end: Iterable[int] = ()) -> Dict[int, torch.Tensor]:
        """push() with the outputs left on the device."""
        x, counts, end = self._pack(chunks, end)
        out = self.push_rows(x, counts, end, host=False)
        return {r: out[r] for r in sorted(set(chunks) | set(end))}

    def save(self, rows) -> torch.Tensor:
        """The rows' state (hop, inputs so far, frames done, last frame's position and tail, history): a uint8
        (len(rows), ROW_BYTES) device tensor."""
        rows = check_rows(rows, self.rows)
        self._check_ready(rows)
        state = torch.empty(len(rows), self.ROW_BYTES, dtype=torch.uint8, device=self.device)
        n = len(rows)
        if n:
            _lib.check(self.lib.q3_stretch_save_rows(self.h, n, (C.c_int32 * n)(*rows), state.data_ptr(), self._stream()))
        return state

    def load(self, rows, state: torch.Tensor):
        """Rows `rows` continue the states save() returned, in order."""
        rows = check_rows(rows, self.rows)
        if not isinstance(state, torch.Tensor) or state.dtype != torch.uint8 \
                or tuple(state.shape) != (len(rows), self.ROW_BYTES) or state.device != self.device:
            raise ValueError(f"expected a saved state of shape ({len(rows)}, {self.ROW_BYTES}) on {self.device}")
        n = len(rows)
        if n == 0:
            return
        state = state.contiguous()
        _lib.check(self.lib.q3_stretch_load_rows(self.h, n, (C.c_int32 * n)(*rows), state.data_ptr(), self._stream()))
        has = state[:, 0:4].cpu().numpy().view(np.int32)[:, 0]   # the header's hop (already read back natively)
        for r, ha in zip(rows, has):
            self._ha[r] = int(ha)

    def oneshot(self, x, speed) -> np.ndarray:
        """The whole clip x (1-D float samples at 24 kHz) stretched at once: the reference of the streamed result."""
        t = check_chunks({0: x}, 1)[0]
        one = TimeStretch(self.device, 1, min(max(t.numel(), 1), self.MAX_IN))
        try:
            one.reset([0], speed)
            return one.push({0: t}, end=[0])[0]
        finally:
            one.close()


class ResampledEncoderStream:
    """An EncoderStream (codec_encoder.py) fed at `sample_rate`: each push goes through a resampler row (sample_rate ->
    the encoder's 24 kHz, float32) on the device into the encoder stream; end(rows) flushes the rows' resampler tails
    into the stream before the encoder's own end, and reset(rows) resets both.  A clip's codes equal
    CodecEncoder.forward of Resampler.oneshot of the clip, bit for bit."""

    def __init__(self, enc, batch: int, max_packet_frames: int, sample_rate: int):
        from .codec_encoder import EncoderStream
        ratio(sample_rate, CODEC_RATE)   # ValueError for an unsupported rate
        self.sample_rate = int(sample_rate)
        self.stream = EncoderStream(enc, batch, max_packet_frames)
        self.batch = self.stream.batch
        self.resampler = Resampler(enc.device, self.batch, int(max_packet_frames) * enc.hop)
        self.resampler.reset(range(self.batch), self.sample_rate, AudioFormat(CODEC_RATE))

    @property
    def positions(self) -> List[int]:
        return self.stream.positions

    def push(self, chunks: Dict) -> Dict[int, torch.Tensor]:
        """{row: 1-D samples at sample_rate} -> {row: (n_i, nq) codes of the frames this push completed}."""
        return self.stream.push(self.resampler.push_device(chunks))

    def end(self, rows) -> Dict[int, torch.Tensor]:
        """End the rows' clips: their resampler tails, then the encoder's last partial frame; returns {row: codes}."""
        rows = check_rows(rows, self.batch)
        if not rows:
            return {}
        codes = self.stream.push(self.resampler.push_device({}, end=rows))
        last = self.stream.end(rows)
        return {r: torch.cat([codes[r], last[r]]) for r in rows}

    def reset(self, rows):
        rows = check_rows(rows, self.batch)
        if not rows:
            return
        self.resampler.reset(rows, self.sample_rate, AudioFormat(CODEC_RATE))
        self.stream.reset(rows)

    def close(self):
        self.stream.close()
        self.resampler.close()
