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

Pitch: a clip time-stretched at 24 kHz and then taken as sampled at 50*Lp Hz (AudioFormat.pitch_step) is resampled
from that rate in one pass: reset / oneshot take such a rate (a multiple of 50 Hz in [12000, 48000]) as in_rate.  The
native table holds MAX_FILTERS filters; each pair's filter is designed on its first use and kept until the table is full
and a new pair needs its entry, when the least recently used pair no row uses is dropped.  save() keeps each row's pair
with its state, so load() adds a dropped filter again.

Speaking rate: TimeStretch, a streaming per-row WSOLA time-stretch at 24 kHz (q3_stretch_*, csrc/stretch.cu, DESIGN
§4.7).  Volume: Limiter, a streaming per-row look-ahead limiter at 24 kHz (q3_limit_*, csrc/limit.cu, DESIGN §4.8).
Loudness: Loudness, a streaming per-row BS.1770 loudness normaliser at 24 kHz (q3_loud_*, csrc/loud.cu, DESIGN §4.9).

The four are row stages (_RowStage) with one streaming contract, and stages(fmt) is the chain of them, in the order
time-stretch, loudness, limiter, resampler, that turns the codec's audio into a client's AudioFormat.
"""
import ctypes as C
from dataclasses import dataclass
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


MAX_FILTERS = 64                   # kMaxFilters: filters a resampler holds at a time
PITCHED_RATES = (12000, 48000)     # the range of 50*Lp, the rate a pitch-shifted clip is resampled from


def ratio(sr_in: int, sr_out: int, pitched: bool = False) -> Tuple[int, int]:
    """(up, down): sr_out / sr_in in lowest terms.  ValueError for a rate outside SUPPORTED_RATES, except that with
    `pitched` sr_in may also be a multiple of 50 Hz in PITCHED_RATES."""
    for sr, alt in ((sr_in, pitched), (sr_out, False)):
        ok = not isinstance(sr, bool) and isinstance(sr, (int, np.integer)) and (
            int(sr) in SUPPORTED_RATES
            or (alt and int(sr) % 50 == 0 and PITCHED_RATES[0] <= int(sr) <= PITCHED_RATES[1]))
        if not ok:
            raise ValueError(f"sample rate {sr!r} is not supported; supported rates: {SUPPORTED_RATES}"
                             + (f", or as input a multiple of 50 Hz in {list(PITCHED_RATES)}" if alt else ""))
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


@dataclass
class ResamplerState:
    """Rows' saved resampler state: the native records (uint8 (n, ROW_BYTES) on the device) and each row's (up, down)
    pair, whose filter may have been dropped and added again under another id by the time the rows are loaded."""
    records: torch.Tensor
    pairs: List[Tuple[int, int]]


def _i32(xs) -> C.Array:
    return (C.c_int32 * len(xs))(*xs)


class _RowStage:
    """`rows` streaming rows of one audio stage on `device` (the native q3_<PREFIX>_* entries), each with its own clip,
    setting and counters.  A push gives each row at most `max_in` samples per launch (longer pushes take several
    launches); output counts follow host formulas, so no push syncs.  reset(rows, ...) starts new clips;
    push({row: samples}, end=rows) returns {row: numpy array of the row's new output}; push_device keeps them on the
    device; save(rows) / load(rows, state) move rows' state; oneshot(x, ...) converts a whole clip with reset's
    settings.  A clip pushed in pieces of any sizes and ended equals oneshot() of the whole clip bit for bit.
    A subclass gives PREFIX, NAME, ROW_BYTES, reset and _max_out."""

    PREFIX = ""                   # the native entries are q3_<PREFIX>_*
    NAME = ""                     # the stage in error messages
    ROW_BYTES = 0                 # one row's saved state
    MAX_IN = 2 ** 31 - 1          # the largest max_in the native stage takes (oneshot pushes in launches of at most it)

    def __init__(self, device, rows: int, max_in: int):
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"{type(self).__name__} needs a CUDA device (no CPU fallback)")
        self.rows, self.max_in = int(rows), int(max_in)
        self.max_out = self._max_out()
        h = C.c_void_p()
        _lib.check(self._fn("open")(self.rows, self.max_in, self.max_out, self.device.index or 0, C.byref(h)))
        self.h = h
        self._enc: List[Optional[str]] = [None] * self.rows   # each row's output encoding; None until reset or loaded
        # every native step writes row r's outputs from byte 4*max_out*r on, in the row's encoding
        self._out = torch.empty(self.rows, 4 * self.max_out, dtype=torch.uint8, device=self.device)
        self._views = {e: self._out.view(dt) for e, dt in _ENC_DTYPE.items()}   # the buffer in each encoding

    def _fn(self, verb: str):
        return getattr(self.lib, f"q3_{self.PREFIX}_{verb}")

    def _max_out(self) -> int:
        """The most outputs one push of max_in inputs plus its end can emit in any setting."""
        raise NotImplementedError

    def close(self):
        if getattr(self, "h", None):
            self._fn("close")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        if not self.h:
            raise RuntimeError(f"{self.NAME} is closed")
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _check_ready(self, rows):
        for r in rows:
            if self._enc[r] is None:
                raise ValueError(f"row {r} was never reset")

    def _reset(self, rows: List[int], *args, enc: str = "f32"):
        """The native reset of the checked `rows` with the per-row arrays `args`; the rows then output `enc`."""
        if rows:
            _lib.check(self._fn("reset_rows")(self.h, len(rows), _i32(rows), *args))
        for r in rows:
            self._enc[r] = enc

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
        enc = {r: self._enc[r] for r in touched}
        st = self._stream()
        parts: Dict[int, list] = {r: [] for r in touched}
        for s0 in range(0, max(max(cnt), 1), self.max_in):
            k = [min(max(c - s0, 0), self.max_in) for c in cnt]
            e = [int(r in end and (s0 == 0 if cnt[r] == 0 else s0 < cnt[r] <= s0 + self.max_in)) for r in range(self.rows)]
            nout = (C.c_int32 * self.rows)()
            ptr = x.data_ptr() + 4 * s0 if x is not None and any(k) else None
            _lib.check(self._fn("step_rows")(self.h, ptr, x.stride(0) if x is not None else 0, _i32(k), _i32(e),
                                             self._out.data_ptr(), nout, st))
            if host:
                nb = {r: nout[r] * _WIDTH[enc[r]] for r in touched}
                top = max(nb.values(), default=0)
                buf = self._out[:, :top].cpu().numpy() if top else None
                for r in touched:
                    parts[r].append(buf[r, :nb[r]].view(_NP_DTYPE[enc[r]]) if nb[r] else None)
            else:
                for r in touched:
                    parts[r].append(self._views[enc[r]][r, :nout[r]].clone() if nout[r] else None)
        out = {}
        for r in touched:
            v = [p for p in parts[r] if p is not None]
            if host:
                out[r] = np.concatenate(v) if v else np.zeros(0, _NP_DTYPE[enc[r]])
            else:
                out[r] = torch.cat(v) if v else torch.zeros(0, dtype=_ENC_DTYPE[enc[r]], device=self.device)
        return out

    def push_rows(self, x: Optional[torch.Tensor], counts: Dict[int, int], end: Iterable[int] = (), host: bool = True):
        """Row r takes x[r, :counts[r]] of x, fp32 (rows, L) on the device with contiguous rows (the layout the codec
        stream returns), and the rows in `end` end their clips: one launch per max_in samples.  Returns {row: its new
        output} (numpy arrays when `host`, else device tensors) for every row with samples or an end and every row of
        `counts`."""
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
        end, in the row's encoding.  One device-to-host copy per launch."""
        x, counts, end = self._pack(chunks, end)
        out = self.push_rows(x, counts, end, host=True)
        return {r: out[r] for r in sorted(set(chunks) | set(end))}

    def push_device(self, chunks: Dict, end: Iterable[int] = ()) -> Dict[int, torch.Tensor]:
        """push() with the outputs left on the device (for an onward stage or the encoder stream)."""
        x, counts, end = self._pack(chunks, end)
        out = self.push_rows(x, counts, end, host=False)
        return {r: out[r] for r in sorted(set(chunks) | set(end))}

    def save(self, rows) -> torch.Tensor:
        """The rows' state: the native records, a uint8 (len(rows), ROW_BYTES) device tensor."""
        rows = check_rows(rows, self.rows)
        self._check_ready(rows)
        state = torch.empty(len(rows), self.ROW_BYTES, dtype=torch.uint8, device=self.device)
        if rows:
            _lib.check(self._fn("save_rows")(self.h, len(rows), _i32(rows), state.data_ptr(), self._stream()))
        return state

    def _fits(self, rec, n: int) -> bool:
        return isinstance(rec, torch.Tensor) and rec.dtype == torch.uint8 and tuple(rec.shape) == (n, self.ROW_BYTES) \
            and rec.device == self.device

    def _records(self, state, n: int) -> torch.Tensor:
        """The records to load from `state`, what save() of n rows returned; ValueError for anything else."""
        if not self._fits(state, n):
            raise ValueError(f"expected a saved state of shape ({n}, {self.ROW_BYTES}) on {self.device}")
        return state.contiguous()

    def load(self, rows, state):
        """Rows `rows` continue the states save() returned, in order."""
        rows = check_rows(rows, self.rows)
        rec = self._records(state, len(rows))
        if not rows:
            return
        _lib.check(self._fn("load_rows")(self.h, len(rows), _i32(rows), rec.data_ptr(), self._stream()))
        self._restore(rows, rec, state)

    def _restore(self, rows: List[int], rec: torch.Tensor, state):
        """The host state of `rows`, just loaded from the records `rec` of `state`."""
        for r in rows:
            self._enc[r] = "f32"

    def oneshot(self, x, *setting, **kw) -> np.ndarray:
        """The whole clip x (1-D float samples) converted at once with reset's `setting`: the reference of the
        streamed result."""
        t = check_chunks({0: x}, 1)[0]
        one = type(self)(self.device, 1, min(max(t.numel(), 1), self.MAX_IN))
        try:
            one.reset([0], *setting, **kw)
            return one.push({0: t}, end=[0])[0]
        finally:
            one.close()


class Resampler(_RowStage):
    """`rows` streaming resampler rows on `device`; a push gives each row at most `max_in` samples per launch (longer
    pushes take several launches).  reset(rows, in_rate, fmt) starts new clips; push({row: samples}, end=rows) returns
    {row: numpy array of the row's new output} in the row's encoding (float32, int16 or uint8); push_device keeps them
    on the device; save(rows) / load(rows, state) move rows' state; release(rows) frees rows' filters for reuse;
    oneshot(x, in_rate, fmt) converts a whole clip."""

    PREFIX, NAME = "resample", "resampler"
    ROW_BYTES = ROW_BYTES

    def __init__(self, device, rows: int, max_in: int):
        super().__init__(device, rows, max_in)
        self._filters: Dict[Tuple[int, int], int] = {}     # pair -> filter id, least recently used first
        self._pair: List[Optional[Tuple[int, int]]] = [None] * self.rows   # the pair each row uses

    def _max_out(self) -> int:
        # capacity for the widest supported pair, so any pair can be added later
        return max(out_bound(self.max_in, *ratio(a, b)) for a in SUPPORTED_RATES for b in SUPPORTED_RATES)

    def _filter(self, up: int, down: int, keep=()) -> int:
        """The id of the pair's filter, designed and added on its first use.  When the table is full, the least
        recently used pair that no row uses and that is not in `keep` is dropped first."""
        pair = (up, down)
        fid = self._filters.pop(pair, None)
        if fid is None:
            if len(self._filters) >= MAX_FILTERS:
                used = set(self._pair) | set(keep)
                old = next((p for p in self._filters if p not in used), None)
                if old is None:
                    raise RuntimeError(f"all {MAX_FILTERS} resampler filters are in use by rows")
                _lib.check(self.lib.q3_resample_drop_filter(self.h, self._filters.pop(old)))
            taps = torch.from_numpy(design(up, down)).to(self.device, torch.float32)
            out = C.c_int32()
            _lib.check(self.lib.q3_resample_add_filter(self.h, up, down, taps.data_ptr(), taps.numel(), C.byref(out)))
            fid = out.value
        self._filters[pair] = fid
        return fid

    def reset(self, rows, in_rate: int, fmt: AudioFormat):
        """Start new clips in `rows` converting in_rate -> fmt.sample_rate into fmt.encoding.  in_rate is a supported
        rate, or a multiple of 50 Hz in PITCHED_RATES (a pitch-shifted clip)."""
        rows = check_rows(rows, self.rows)
        fmt = check_format(fmt)
        pair = ratio(in_rate, fmt.sample_rate, pitched=True)
        fid = self._filter(*pair)
        n = len(rows)
        self._reset(rows, _i32([fid] * n), _i32([_ENC_CODE[fmt.encoding]] * n), enc=fmt.encoding)
        for r in rows:
            self._pair[r] = pair

    def release(self, rows):
        """Rows `rows` no longer use their filters (which may then be dropped); they need a reset or a load before
        their next push."""
        rows = check_rows(rows, self.rows)
        if rows:
            _lib.check(self.lib.q3_resample_release_rows(self.h, len(rows), _i32(rows)))
        for r in rows:
            self._enc[r] = self._pair[r] = None

    def save(self, rows) -> ResamplerState:
        """The rows' state: the native records (filter, encoding, inputs so far, history; a uint8 (len(rows),
        ROW_BYTES) device tensor) with each row's rate pair."""
        rows = check_rows(rows, self.rows)
        return ResamplerState(super().save(rows), [self._pair[r] for r in rows])

    def _records(self, state, n: int) -> torch.Tensor:
        # a pair whose filter was dropped since the save is added again, and the records get each pair's current id
        if not isinstance(state, ResamplerState) or not self._fits(state.records, n) or len(state.pairs) != n:
            raise ValueError(f"expected a ResamplerState of {n} rows on {self.device}")
        fids = [self._filter(*p, keep=state.pairs) for p in state.pairs]
        rec = state.records.clone()
        rec[:, 0:4] = torch.tensor(fids, dtype=torch.int32).view(torch.uint8).reshape(n, 4).to(self.device)
        return rec

    def _restore(self, rows, rec, state):
        codes = rec[:, 4:8].cpu().numpy().view(np.int32)[:, 0]   # the header's encoding (already read back natively)
        for r, c, p in zip(rows, codes, state.pairs):
            self._enc[r], self._pair[r] = ENCODINGS[c], p


class TimeStretch(_RowStage):
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
    PREFIX, NAME = "stretch", "time-stretch"
    ROW_BYTES = 10144                 # Q3_STRETCH_ROW_BYTES: one row's saved state
    MAX_IN = 32768                    # the largest max_in the native stretcher takes

    @staticmethod
    def hop(speed, pitch=0.0) -> int:
        """The analysis hop of `speed` at `pitch` semitones (AudioFormat.hop): floor(speed*480*(480/Lp) + 0.5), which
        is floor(speed*480 + 0.5) at pitch 0; the effective speed is hop*Lp/480^2.  ValueError outside AudioFormat's
        ranges, or for a hop outside [240, 960]."""
        return AudioFormat(CODEC_RATE, speed=speed, pitch=pitch).hop

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
        super().__init__(device, rows, max_in)
        w = torch.from_numpy(self.window()).to(self.device, torch.float32)
        _lib.check(self.lib.q3_stretch_set_window(self.h, w.data_ptr()))

    def _max_out(self) -> int:
        if not 1 <= self.max_in <= self.MAX_IN:
            raise ValueError(f"max_in {self.max_in} outside [1, {self.MAX_IN}]")
        return self.out_bound(self.max_in)

    def reset(self, rows, speed, pitch=0.0):
        """Start new clips in `rows` at `speed` and `pitch` (analysis hop hop(speed, pitch))."""
        rows = check_rows(rows, self.rows)
        ha = self.hop(speed, pitch)
        self._reset(rows, _i32([ha] * len(rows)))


class Limiter(_RowStage):
    """`rows` streaming look-ahead limiter rows at the codec's 24 kHz on `device` (q3_limit_*, csrc/limit.cu, DESIGN
    §4.8): a gain of `volume` dB whose peaks are held at -1 dBFS, with 5 ms of look-ahead and a linear release of at most
    50 ms.  A clip of n samples gives n samples; after n samples without an end a row has emitted emitted(n) = max(0,
    n - 119), so the limiter delays by 119 samples.  A push gives each row at most `max_in` samples per launch (longer
    pushes take several launches).  reset(rows, volume) starts new clips; push({row: samples}, end=rows) returns {row:
    float32 numpy array of the row's new output}; push_device keeps them on the device; save(rows) / load(rows, state)
    move rows' state; oneshot(x, volume) limits a whole clip.  A clip pushed in pieces of any sizes and ended equals
    oneshot() of the whole clip bit for bit."""

    L, W = 120, 1200                  # look-ahead, release
    DELAY = L - 1
    HIST = 1536                       # Q3_LIMIT_HIST: inputs a row keeps (it reads W + 2L - 2 = 1438 back)
    PREFIX, NAME = "limit", "limiter"
    ROW_BYTES = 6160                  # Q3_LIMIT_ROW_BYTES: one row's saved state

    @staticmethod
    def gain(volume) -> np.float32:
        """fp32(10^(volume/20)), designed in fp64.  ValueError outside AudioFormat's volume range."""
        return np.float32(10.0 ** (AudioFormat(CODEC_RATE, volume=volume).volume / 20))

    @classmethod
    def emitted(cls, n: int) -> int:
        """Outputs a row has emitted after n inputs without an end: max(0, n - 119)."""
        return max(0, n - cls.DELAY)

    @staticmethod
    def total(n: int) -> int:
        """Outputs of a whole clip of n inputs: n."""
        return n

    def _max_out(self) -> int:
        return self.max_in + self.DELAY

    def reset(self, rows, volume):
        """Start new clips in `rows` at `volume` dB (gain gain(volume))."""
        rows = check_rows(rows, self.rows)
        g = self.gain(volume)
        self._reset(rows, (C.c_float * len(rows))(*[g] * len(rows)))


class Loudness(_RowStage):
    """`rows` streaming loudness normaliser rows at the codec's 24 kHz on `device` (q3_loud_*, csrc/loud.cu, DESIGN
    §4.9): a gain towards a target integrated loudness in LUFS, measured while the audio streams.  The input is K-weighted
    (k_weighting(), BS.1770-4) over 100 ms segments; when a segment completes, the gated loudness of the clip so far
    (blocks of the last four segments, the -70 LUFS and -10 LU gates) gives the gain A_s = 10^(clamp(target - I_s, -30,
    30)/20), and the samples of segment k ramp linearly from A_{k-2} to A_{k-1}.  So the first 100 ms pass at unity gain,
    silence holds the last gain, and there is no delay: a clip of n samples gives n samples, emitted(n) = n.  A clip may
    hold at most MAX_BLOCKS segments.  A push gives each row at most `max_in` samples per launch (longer pushes take
    several launches).  reset(rows, target) starts new clips; push({row: samples}, end=rows) returns {row: float32 numpy
    array of the row's new output}; push_device keeps them on the device; save(rows) / load(rows, state) move rows'
    state; oneshot(x, target) normalises a whole clip.  A clip pushed in pieces of any sizes and ended equals oneshot()
    of the whole clip bit for bit.  A raised gain can clip: the batcher always runs the Limiter after it."""

    SEG = 2400                        # samples per segment (100 ms)
    MAX_BLOCKS = 16384                # Q3_LOUD_MAX_BLOCKS: segments one clip may hold (27 min 18.4 s)
    PREFIX, NAME = "loud", "loudness normaliser"
    ROW_BYTES = 140736                # Q3_LOUD_ROW_BYTES: one row's saved state
    MAX_IN = 32768                    # the largest max_in the native stage takes

    @staticmethod
    def k_weighting(fs: int = CODEC_RATE) -> np.ndarray:
        """The BS.1770-4 K-weighting at `fs` as fp64 second-order sections (2, 6), rows b0 b1 b2 a0 a1 a2: the shelf,
        then the high-pass, by libebur128's bilinear design (uploaded as fp32)."""
        def section(f0, q, vh, vb):
            k = np.tan(np.pi * f0 / fs)
            a0 = 1 + k / q + k * k
            a = [1.0, 2 * (k * k - 1) / a0, (1 - k / q + k * k) / a0]
            if vh is None:
                return [1.0, -2.0, 1.0] + a
            return [(vh + vb * k / q + k * k) / a0, 2 * (k * k - vh) / a0, (vh - vb * k / q + k * k) / a0] + a
        vh = 10 ** (3.999843853973347 / 20)
        return np.array([section(1681.974450955533, 0.7071752369554196, vh, vh ** 0.4996667741545416),
                         section(38.13547087602444, 0.5003270373238773, None, None)])

    @staticmethod
    def emitted(n: int) -> int:
        """Outputs a row has emitted after n inputs without an end: n."""
        return n

    @staticmethod
    def total(n: int) -> int:
        """Outputs of a whole clip of n inputs: n."""
        return n

    def __init__(self, device, rows: int, max_in: int):
        super().__init__(device, rows, max_in)
        sos = self.k_weighting().astype(np.float32).ravel()
        _lib.check(self.lib.q3_loud_set_filter(self.h, (C.c_float * 12)(*sos)))

    def _max_out(self) -> int:
        if not 1 <= self.max_in <= self.MAX_IN:
            raise ValueError(f"max_in {self.max_in} outside [1, {self.MAX_IN}]")
        return self.max_in

    def reset(self, rows, target):
        """Start new clips in `rows` normalised towards `target` LUFS (AudioFormat's loudness range)."""
        rows = check_rows(rows, self.rows)
        t = AudioFormat(CODEC_RATE, loudness=target).loudness
        self._reset(rows, (C.c_double * len(rows))(*[t] * len(rows)))


STAGES = ("TimeStretch", "Loudness", "Limiter", "Resampler")   # the stage classes above, in the order a stream runs them


def stages(fmt: Optional[AudioFormat]) -> Tuple[Tuple[str, tuple], ...]:
    """The stages the codec's audio runs through to come out in `fmt`, in STAGES order, each as (its class's name in
    this module, the arguments its reset takes after the rows): the time-stretch when the hop is not 480, (speed, pitch)
    when the pitch step Lp is not 480 and (speed,) (pitch 0) when it is; the loudness normaliser (loudness,) with a
    loudness target; the limiter (volume,) at a volume other than 0 dB, and always after a loudness target; the resampler (50*Lp, AudioFormat(rate, encoding)) when Lp is not 480 or the rate or encoding is not 24 kHz
    float32.  () for None (the codec's own audio)."""
    if fmt is None:
        return ()
    fmt = check_format(fmt)
    pitched = fmt.pitch_step != 480
    out = AudioFormat(fmt.sample_rate, fmt.encoding)
    chain = []
    if fmt.hop != 480:
        chain.append(("TimeStretch", (fmt.speed, fmt.pitch) if pitched else (fmt.speed,)))
    if fmt.loudness is not None:
        chain.append(("Loudness", (fmt.loudness,)))
    if fmt.volume != 0 or fmt.loudness is not None:
        chain.append(("Limiter", (fmt.volume,)))
    if pitched or out != AudioFormat(CODEC_RATE):
        chain.append(("Resampler", (50 * fmt.pitch_step, out)))
    return tuple(chain)


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
