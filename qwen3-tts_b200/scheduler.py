"""Continuous batching over the AR engine (SURVEY §8f-4).

The reference serves one static, left-padded batch per `generate()` call (modeling_qwen3_tts.py:2239-2254) behind a
Gradio queue (cli/demo.py:629): a request that arrives while a batch is running waits for the whole batch, and a
batch runs until its LONGEST utterance ends.  Here a session of `n_slots` rows runs continuously; a request is
prefilled into a free slot between two decode chunks (`packet_frames` frame-steps) while the other rows keep their
K/V, positions, sampling history and Philox streams, and leaves as soon as it samples EOS.  Every per-row quantity of
the fused kernel is keyed by the row's own frame counter and by the request's Philox key, so a request generates
exactly what it would generate alone (tests/test_gpu_scheduler.py).

Each request may carry its own SamplingParams (greedy or sampled, temperature, top-k / top-p, repetition penalty,
min_new_tokens, the subtalker's settings, the Philox seed): the kernel reads every sampling field from the row's own
entry, so requests with different parameters share one session, and each still generates what it would alone in a
session whose default is its parameters (tests/test_gpu_scheduler_sampling.py).  Slots without a running request
sample with the session's parameters.

With a codec the batcher also streams audio: one codec stream of `n_slots` rows follows the session, a slot's row is
reset when a request enters it, and after every decode each running slot pushes its new frames as its own count (idle
slots push none).  A request's concatenated chunks equal the one-shot decode of its codes alone
(tests/test_gpu_scheduler_audio.py).  `packets()` hands out the new codes instead, for callers that decode them
themselves.  TTSEngine.stream_synthesize runs its static batch as such a session: B requests submitted together are
admitted in one call, in slots and with Philox keys 0..B-1, which is what q3_prefill does.

A request may carry reference codes (voice cloning, `ref_codes` of submit): the reference decodes cat(ref_code,
generated codes) and cuts the reference's audio off (qwen3_tts_model.py:612-631), so the generated frames are decoded
with the reference as their causal left context.  At admission such a slot's codec row is seeded with its reference
(CodecStream.seed, one call for all seeded slots of the admission) instead of reset; its chunks and `done` entry hold
the generated part only (tests/test_gpu_scheduler_voice_clone.py).

A request of a registered voice (`submit(suffix, trailing, voice=voice)`, Qwen3TTSModel.register_voice) is admitted
with the voice's prompt prefix: its K/V are copied into the slot (AREngine.admit(..., prefixes=)) and only the
request's own rows are prefilled, and an ICL voice's codec row is copied from the decoder's reference bank
(CodecStream.copy_from, one call per bank) instead of decoding the reference.  It generates and streams exactly what
the request submitted with its whole prompt and ref_codes does (tests/test_gpu_voice_prefix.py).  A batch without
voices makes the same calls as before.

Live text (`submit(text_open=True)`, `append_text`, `close_text`): a request's text may keep arriving after submit, as
when speaking an LLM's answer while it is being written.  Its slot is open in the engine (AREngine.set_text_open): a
frame-step whose text row has not arrived holds the row instead of reading tts_pad, so the request generates exactly
what it generates with the whole text given up front (tests/test_gpu_live_text.py).  A step launches only when it
admits a request or some running row can produce a frame: a closed row always can, an open row when its text reaches
the frames it has reported.  Otherwise the step launches nothing and returns no frames, and `stream()` / `packets()`
yield empty results, so a single-threaded caller feeds text between iterations.  `cancel` drops a request, pending or
running (a client that disconnected).

Parking: a running request can leave its slot and continue later in any free slot (AREngine.park / resume): its talker
K/V and row state wait in an engine record, its codes so far on the request, its codec row in a row of the decoder's
bank (CodecDecoder.bank_copy), so it generates and streams exactly what it would have never parked
(tests/test_gpu_park.py).  `park(rid)` / `resume(rid)` do this on request, for example for a client that stopped
reading.  With `park_waiting=True` the batcher parks live-text requests that wait for text whenever a pending or a
resumable parked request needs a slot and none is free, and resumes them once their text covers their next frame.
Each step parks first, then resumes parked requests into free slots (oldest park first, ahead of admissions), then
admits.

Live text of an ICL voice clone (`submit(..., text_open=True, overlay=)`, Qwen3TTSModel.build_live_clone_request): the
last positions of its prompt overlay reference codes with target text, one text row each, so its prompt is complete
only once that many text rows have arrived.  Text rows fill the overlay first (row i of the prompt becomes overlay[i] +
text row, the bf16 add of build_prefill), later rows are trailing text; a close_text before the overlay is full
completes it with tts_pad and makes the trailing text [tts_pad], build_prefill's layout for a short text.  Until then
the request is not admitted, takes no slot a park would free, and does not keep run() going; once complete it is
admitted and runs as any live request, so it generates what its whole text gives up front (tests/test_gpu_live_clone.py).

Audio formats (`ContinuousBatcher(audio_format=)` for the session, `submit(audio_format=)` per request, an AudioFormat
of rate, encoding, speed, pitch, volume and loudness): a request's audio runs through the chain of stages audio.stages
gives its format, in order a time-stretch (a speed or pitch), a loudness normaliser (a loudness target), a limiter (a
volume, or a loudness target) and a resampler (a pitch, or a rate or encoding other than 24 kHz float32); a request in
the codec's own format has none.  Each stage is one object of
`n_slots` rows, opened when the first request that uses it is admitted, and a request has a row in each stage of its
chain, in its slot.  The rows are reset at admission after the codec row's reset, seed or bank copy (they shape the
generated part only), one reset per stage and setting; saved on the request when it is parked, loaded into its new
slot when it is resumed, and dropped with it on cancel.  After each codec push one launch per stage serves every slot
that uses it, the samples going from stage to stage on the device; a request that finished in the step ends its row in
each stage, so each stage's tail goes on into the next stage's end in the same step (even with no new frame), and
stream() yields its chunk as float32, int16 or uint8.  A request's concatenated chunks equal
    Resampler.oneshot(Limiter.oneshot(Loudness.oneshot(TimeStretch.oneshot(w, speed, pitch), target), volume), 50*Lp,
                      AudioFormat(rate, encoding))
bit for bit, w its whole waveform, Lp its pitch step and each stage skipped when its chain has none
(tests/test_gpu_scheduler_audio_format.py, test_gpu_scheduler_speed.py, test_gpu_scheduler_pitch_volume.py,
test_gpu_scheduler_loudness.py).  A loudness request whose longest possible audio (its horizon's samples, stretched)
passes Loudness.MAX_BLOCKS segments is refused at submit.  A session without formats opens no stage and makes the
same calls as before.
"""
from collections import deque
from dataclasses import dataclass, field
from typing import Any, Deque, Dict, Iterator, List, Optional, Tuple, Union

import numpy as np
import torch

from . import audio
from .codec import CodecDecoder, CodecStream, check_ref_codes
from .config import AudioFormat, SamplingParams
from .engine import AREngine


@dataclass
class _Request:
    rid: int
    embeds: torch.Tensor
    trailing: torch.Tensor
    max_frames: int
    sampling: Optional[SamplingParams] = None
    ref_codes: Optional[torch.Tensor] = None
    voice: Optional[Any] = None   # a registered voice (model.Voice): its prompt prefix and reference state
    text_open: bool = False    # submitted with text that may still grow
    closed: bool = False       # close_text() was called
    n_text: int = 0            # trailing rows given so far (`trailing`: those the engine does not have yet)
    slot: int = -1
    emitted: int = 0
    chunks: List[torch.Tensor] = field(default_factory=list)
    paused: bool = False       # park(rid) without resume(rid): not admitted, parked at the next step, not resumed
    record: int = -1           # while parked: the engine's record, the codec bank row and the codes so far
    bank: Optional[Tuple[int, int]] = None
    codes: Optional[torch.Tensor] = None
    overlay: Optional[torch.Tensor] = None   # prompt rows still waiting for a text row each (None once complete)
    chain: Dict[str, tuple] = field(default_factory=dict)   # its stages in order: {name: reset arguments} (audio.stages)
    saved: Dict[str, Any] = field(default_factory=dict)     # while parked: {stage name: its row's saved state}
    # while parked: its row's saved state in each stage, None without a row there
    st_state = property(lambda self: self.saved.get("TimeStretch"))
    loud_state = property(lambda self: self.saved.get("Loudness"))
    lim_state = property(lambda self: self.saved.get("Limiter"))
    res_state = property(lambda self: self.saved.get("Resampler"))

    @property
    def shaped(self) -> bool:
        """Its audio goes through a chain of stages."""
        return bool(self.chain)


class ContinuousBatcher:
    def __init__(self, engine: AREngine, tts_pad_embed: torch.Tensor, sp: SamplingParams, n_slots: int = 8, packet_frames: int = 4,
                 max_trailing: int = 256, codec: Union[CodecDecoder, CodecStream, None] = None, park_waiting: bool = False,
                 audio_format: Optional[AudioFormat] = None):
        """`codec`: a CodecDecoder, whose stream of `n_slots` rows the batcher opens, or an open CodecStream of
        `n_slots` rows taking packets of at least `packet_frames` frames.  `park_waiting`: park running live-text
        requests that wait for text when another request needs their slot (see the module docstring).
        `audio_format`: the sample rate and encoding of stream()'s audio for requests submitted without one (None:
        the codec's 24 kHz float32)."""
        self.eng, self.sp, self.pad = engine, sp, tts_pad_embed
        self.park_waiting = bool(park_waiting)
        self.parked: Dict[int, _Request] = {}      # request id -> parked request, oldest park first
        self.moves: List[Tuple[str, int, int]] = []   # ("park" | "resume", request id, slot), in order
        self.n_slots, self.packet = int(n_slots), int(packet_frames)
        self.G = engine.cfg.num_code_groups
        self.max_frames = max(int(sp.max_new_tokens) - 1, 1)
        self.codes = torch.zeros(self.n_slots, self.max_frames, self.G, dtype=torch.int32, device=engine.device)
        self.pending: Deque[_Request] = deque()
        self.running: Dict[int, _Request] = {}     # slot -> request
        self.done: Dict[int, torch.Tensor] = {}
        self._next_id = 0
        self._cancelled = set()
        self.max_trailing = int(max_trailing)
        engine.session_begin(self.n_slots, tts_pad_embed, sp, max_trailing=self.max_trailing)
        self.frames_total = 0
        if isinstance(codec, CodecStream):
            if codec.B != self.n_slots or codec.nmax < self.packet:
                raise ValueError(f"a codec stream of {codec.B} rows and packets of up to {codec.nmax} frames cannot "
                                 f"serve {self.n_slots} slots with packets of {self.packet} frames")
            self.codec, self.cstream = codec.dec, codec
        elif codec is None or hasattr(codec, "open_stream"):   # a CodecDecoder (or a test's stand-in for one)
            self.codec = codec
            self.cstream = codec.open_stream(self.n_slots, max_packet_frames=self.packet) if codec is not None else None
        else:
            raise ValueError(f"codec must be a CodecDecoder or a CodecStream, got {type(codec).__name__}")
        self._chain(audio_format)
        self.audio_format = audio_format
        self.stages: Dict[str, Any] = {}   # stage name -> its object, in chain order; opened by the first request using it

    # each stage of `stages`, None until the first request that uses it is admitted
    stretcher = property(lambda self: self.stages.get("TimeStretch"))
    loudness = property(lambda self: self.stages.get("Loudness"))
    limiter = property(lambda self: self.stages.get("Limiter"))
    resampler = property(lambda self: self.stages.get("Resampler"))

    def _chain(self, fmt: Optional[AudioFormat]) -> Dict[str, tuple]:
        """The stages a request in `fmt` runs, in order, with their reset arguments (audio.stages)."""
        chain = dict(audio.stages(fmt))
        if fmt is not None and self.codec is None:
            raise ValueError("an audio format needs a ContinuousBatcher built with a codec")
        return chain

    def _stage(self, name: str):
        """The stage `name` (a class of audio, looked up when it is opened, on first use), kept in chain order."""
        if name not in self.stages:
            self.stages[name] = getattr(audio, name)(self.eng.device, self.n_slots, self.packet * self.codec.total_upsample)
            self.stages = {n: self.stages[n] for n in audio.STAGES if n in self.stages}
        return self.stages[name]

    # ------------------------------------------------------------------ API
    def submit(self, inputs_embeds: torch.Tensor, trailing_text: Optional[torch.Tensor] = None, key: Optional[int] = None,
               max_frames: Optional[int] = None, sampling: Optional[SamplingParams] = None,
               ref_codes: Optional[torch.Tensor] = None, text_open: bool = False, voice=None,
               overlay: Optional[torch.Tensor] = None, audio_format: Optional[AudioFormat] = None) -> int:
        """Queue one request; returns its id (also its Philox row key unless `key` is given).  `sampling`: the
        request's own generation parameters (default: the session's); its max_new_tokens bounds the request's horizon
        and may not exceed the session's.  `ref_codes`: (L, num_quantizers) reference codes of a voice-clone request
        (VoiceClonePromptItem.ref_code); its audio is decoded after them, and the horizon leaves the codec's RoPE
        table room for them.  `text_open`: the request's text may grow after submit (append_text, then close_text);
        until it is closed the request waits for text instead of reading tts_pad past its end.  `voice`: a registered
        voice (Qwen3TTSModel.register_voice) of this engine, and of this codec if it clones with a reference; the prompt
        is then the voice's prefix followed by `inputs_embeds` (the suffix of Qwen3TTSModel.build_voice_request), the
        prefix's K/V are copied at admission instead of prefilled, and an ICL voice's codec row is copied from its
        reference state instead of decoding the reference.  It takes no `ref_codes`.  `overlay`: (K, H) prompt rows of
        a live ICL voice clone that still wait for one text row each (Qwen3TTSModel.build_live_clone_request); it needs
        `text_open`, and an ICL voice if it has a voice.  The trailing rows given here and later fill it first, and the
        request is admitted once it is full or its text is closed (see the module docstring).  `audio_format`: the
        sample rate and encoding of the request's stream() chunks (default: the session's).  Bad parameters raise
        ValueError here, never in a later step()."""
        chain = self._chain(audio_format if audio_format is not None else self.audio_format)
        H = self.eng.cfg.talker.hidden_size
        L_ref, P = 0, 0
        if overlay is not None:
            if not text_open:
                raise ValueError("an overlay waits for text: submit it with text_open=True")
            if overlay.dim() != 2 or overlay.shape[1] != H:
                raise ValueError(f"overlay must be a (K, {H}) tensor, got {tuple(overlay.shape)}")
            if voice is not None and (not voice.icl or voice.non_streaming_mode):
                raise ValueError("an overlay belongs to an ICL voice registered with non_streaming_mode=False")
            if self.max_trailing < 1:
                raise ValueError("an overlay may end in a tts_pad trailing row: it needs max_trailing >= 1")
        if voice is not None:
            if ref_codes is not None:
                raise ValueError("a registered voice carries its own reference: submit it without ref_codes")
            if voice.closed:
                raise ValueError("the voice is closed")
            if voice.engine is not self.eng:
                raise ValueError("the voice was registered on another engine")
            if voice.bank is not None and (self.codec is None or voice.codec is not self.codec):
                raise ValueError("the voice's reference state belongs to another codec")
            P = voice.prefix_len
            L_ref = voice.ref_len if self.codec is not None else 0
        if ref_codes is not None:
            if self.codec is None:
                raise ValueError("ref_codes need a ContinuousBatcher built with a codec")
            L_ref = check_ref_codes(self.codec.cfg, ref_codes, self.codec.max_frames - 1, "ref_codes")
        limit = self.max_frames   # frames the request may generate: HF emits max_new_tokens - 1 complete frames
        if sampling is not None:
            self.eng.check_sampling(sampling)
            want = int(sampling.max_new_tokens) - 1
            if want > self.max_frames:
                raise ValueError(f"max_new_tokens={sampling.max_new_tokens} exceeds the session's "
                                 f"max_new_tokens={self.sp.max_new_tokens} (its codes buffer holds {self.max_frames} frames)")
            limit = max(want, 0)
        rid = self._next_id if key is None else int(key)
        self._next_id = max(self._next_id, rid) + 1
        tr = trailing_text if trailing_text is not None else torch.zeros(0, H)
        K = 0 if overlay is None else int(overlay.shape[0])
        if max(tr.reshape(-1, H).shape[0] - K, 0) > self.max_trailing:
            raise ValueError(f"trailing text of {tr.shape[0]} positions exceeds max_trailing={self.max_trailing}")
        S = int(inputs_embeds.reshape(-1, H).shape[0])
        if voice is not None and S + K < 1:
            raise ValueError("a request of a registered voice needs at least one row of its own")
        L = P + S + K
        room = self.eng.max_ctx - L
        if room < 1:
            raise ValueError(f"prompt of {L} positions does not fit max_ctx={self.eng.max_ctx}")
        horizon = min(limit if max_frames is None else max_frames, limit, room)
        if self.codec is not None:
            horizon = min(horizon, self.codec.max_frames - L_ref)  # a codec row's position may not pass its RoPE table
        if "Loudness" in chain:
            fmt = audio_format if audio_format is not None else self.audio_format
            n = audio.TimeStretch.total(horizon * self.codec.total_upsample, fmt.hop)
            if n > audio.Loudness.MAX_BLOCKS * audio.Loudness.SEG:
                raise ValueError(f"a loudness target measures at most {audio.Loudness.MAX_BLOCKS} segments of "
                                 f"{audio.Loudness.SEG} samples, and this request may stream {n} samples: lower "
                                 f"max_frames")
        r = _Request(rid, inputs_embeds, tr, horizon, sampling, ref_codes, voice, text_open=bool(text_open),
                     overlay=overlay if K else None, chain=chain)
        if r.overlay is not None:
            r.trailing = self._fill(r, tr.reshape(-1, H))
        r.n_text = int(r.trailing.reshape(-1, H).shape[0])
        self.pending.append(r)
        if voice is not None:
            voice.pending += 1
        return rid

    def _find(self, rid: int, what: str) -> _Request:
        """The pending, running or parked request `rid`, else ValueError."""
        r = next((q for q in self.pending if q.rid == rid), None) or next((q for q in self.running.values() if q.rid == rid), None) \
            or self.parked.get(rid)
        if r is None:
            state = "was cancelled" if rid in self._cancelled else "has finished" if rid in self.done else "is unknown"
            raise ValueError(f"{what}: request {rid} {state}")
        return r

    def _live(self, rid: int, what: str) -> _Request:
        """The pending, running or parked request `rid` whose text is still open, else ValueError."""
        r = self._find(rid, what)
        if not r.text_open:
            raise ValueError(f"{what}: request {rid} was not submitted with text_open=True")
        if r.closed:
            raise ValueError(f"{what}: the text of request {rid} is already closed")
        return r

    def append_text(self, rid: int, rows: torch.Tensor):
        """More trailing text rows (n, H) for an open request, pending, running or parked (Qwen3TTSModel.live_text_rows makes
        them from a piece of text).  ValueError for an unknown, finished or cancelled request, one that was not
        submitted open or is already closed, or text beyond max_trailing."""
        r = self._live(rid, "append_text")
        H = self.eng.cfg.talker.hidden_size
        rows = rows.reshape(-1, H)
        n = rows.shape[0] - (0 if r.overlay is None else min(r.overlay.shape[0], rows.shape[0]))
        if r.n_text + n > self.max_trailing:
            raise ValueError(f"append_text: request {rid} would have {r.n_text + n} trailing rows, more than "
                             f"max_trailing={self.max_trailing}")
        if r.overlay is not None:
            rows = self._fill(r, rows)
        if rows.shape[0] == 0:
            return
        if r.slot >= 0:
            self.eng.append_trailing(r.slot, rows)
        else:
            r.trailing = torch.cat([r.trailing.reshape(-1, H).to(rows.device, rows.dtype), rows], 0)
        r.n_text += int(rows.shape[0])

    def close_text(self, rid: int):
        """No more text is coming for `rid` (append Qwen3TTSModel.live_text_end() first): past its text the request
        reads tts_pad and ends.  ValueError as for append_text."""
        r = self._live(rid, "close_text")
        r.closed = True
        if r.overlay is not None:   # the text ended inside the overlay: build_prefill's layout of a short text
            pad = self.pad.reshape(1, -1)
            self._fill(r, pad.expand(r.overlay.shape[0], -1))
            r.trailing, r.n_text = pad, 1
        if r.slot >= 0:
            self.eng.set_text_open(r.slot, False)

    def _fill(self, r: _Request, rows: torch.Tensor) -> torch.Tensor:
        """Text rows (n, H) of pending request r go to its overlay first: each completes the next waiting prompt row
        (overlay row + text row, in bf16 as build_prefill adds them).  Returns the rows left over, trailing text."""
        m = min(r.overlay.shape[0], rows.shape[0])
        if m:
            done = r.overlay[:m] + rows[:m].to(r.overlay.device, r.overlay.dtype)
            r.embeds = torch.cat([r.embeds.reshape(-1, done.shape[1]).to(done.device, done.dtype), done], 0)
            r.overlay = r.overlay[m:] if m < r.overlay.shape[0] else None
        return rows[m:]

    def cancel(self, rid: int) -> bool:
        """Drop request `rid`: a pending one leaves the queue, a running one's slot is released (its codec row is reset
        at the slot's next admission).  It gets no `done` entry.  False when there is no such pending or running
        request."""
        for r in self.pending:
            if r.rid == rid:
                self.pending.remove(r)
                if r.voice is not None:
                    r.voice.pending -= 1
                self._cancelled.add(rid)
                return True
        for slot, r in self.running.items():
            if r.rid == rid:
                self.eng.release_slots([slot])
                del self.running[slot]
                self._cancelled.add(rid)
                return True
        r = self.parked.pop(rid, None)
        if r is not None:    # its record, its codec bank row and its stages' states are freed
            self.eng.discard(r.record)
            if r.bank is not None:
                self.codec.bank_release(*r.bank)
            r.saved = {}
            self._cancelled.add(rid)
            return True
        return False

    def park(self, rid: int):
        """Take request `rid` out of its slot until resume(rid): a running request is parked at the next step boundary
        (its slot is then free for others), a pending one is not admitted.  ValueError for an unknown, finished or
        cancelled request."""
        self._find(rid, "park").paused = True

    def resume(self, rid: int):
        """Make a request of park(rid) eligible again: a parked one is resumed into the next free slot (a live-text
        request once its text covers its next frame), a pending one may be admitted, a running one stays.  ValueError as
        for park."""
        self._find(rid, "resume").paused = False

    def _waiting(self, r: _Request) -> bool:
        """An open live-text request whose text does not cover its next frame (the negation of _runnable's test)."""
        return r.text_open and not r.closed and r.n_text < r.emitted

    def _resumable(self, r: _Request) -> bool:
        return not r.paused and not self._waiting(r)

    @staticmethod
    def _admissible(r: _Request) -> bool:
        """A pending request that may take a slot: not paused, and its prompt complete (no overlay waits for text)."""
        return not r.paused and r.overlay is None

    def _park(self, slot: int):
        """Park the running request of `slot`: its engine row into a record, its codes so far onto the request, its codec
        row into a bank row."""
        r = self.running.pop(slot)
        r.codes = self.codes[slot, :r.emitted].clone()
        r.record = self.eng.park(slot)
        if self.cstream is not None:
            r.bank = self.codec.bank_copy(self.cstream, slot)
        r.saved = {name: self.stages[name].save([slot]) for name in r.chain}
        r.trailing = r.trailing.reshape(-1, self.eng.cfg.talker.hidden_size)[:0]   # the record holds the text so far
        r.slot = -1
        self.parked[r.rid] = r
        self.moves.append(("park", r.rid, slot))

    def _resume(self, r: _Request, slot: int):
        """Put parked request r into the free slot `slot`: the engine row, its codes, its codec row, the text that
        arrived while it was parked and its live-text state."""
        self.eng.resume(r.record, slot)
        del self.parked[r.rid]
        r.record, r.slot = -1, slot
        self.running[slot] = r
        if r.emitted > 0:
            self.codes[slot, :r.emitted] = r.codes
        r.codes = None
        if r.bank is not None:
            self.cstream.copy_from(self.codec.bank_stream(r.bank[0]), [r.bank[1]], [slot])
            self.codec.bank_release(*r.bank)   # a later bank_copy into that row is queued behind this copy
            r.bank = None
        for name, state in r.saved.items():
            self.stages[name].load([slot], state)
        r.saved = {}
        if r.trailing.shape[0] > 0:
            self.eng.append_trailing(slot, r.trailing)
            r.trailing = r.trailing[:0]
        if r.text_open:
            self.eng.set_text_open(slot, not r.closed)
        self.moves.append(("resume", r.rid, slot))

    def step(self) -> List[int]:
        """Admit what fits, decode one packet, collect what finished.  Returns the ids that completed in this step."""
        new, finished = self._advance()
        self._push_audio(new)
        return finished

    def stream(self) -> Iterator[Tuple[Dict[int, np.ndarray], List[int]]]:
        """Run the session with audio out: yields per step ({request id: waveform of its new frames},
        [ids that finished in the step]) while requests are pending, running or parked, so a request submitted between
        two iterations is admitted at the next one.  A waveform is float32 at the codec's 24 kHz, or in the request's
        audio format (float32, int16 or uint8 at its rate); a request with a format also gets an entry in the step it
        finishes, holding its stages' tails."""
        if self.cstream is None:
            raise ValueError("stream() needs a ContinuousBatcher built with a codec")
        while self.pending or self.running or self.parked:
            new, finished = self._advance()
            yield self._push_audio(new), finished

    def packets(self) -> Iterator[Tuple[Dict[int, torch.Tensor], List[int]]]:
        """Run the session with codes out: yields per step ({request id: (k, G) int64 codes of its k new frames},
        [ids that finished in the step]) while requests are pending, running or parked.  The codec stream, if any, is
        not pushed."""
        while self.pending or self.running or self.parked:
            new, finished = self._advance()
            yield {r.rid: self.codes[slot, e0:e0 + k].to(torch.int64) for slot, (r, e0, k) in new.items() if k > 0}, finished

    def _runnable(self) -> bool:
        """Some running row can produce a frame in the next launch: a closed row always can; an open row when its
        text covers the frames it has reported (the step after them has its text row, or is the one held step that
        completes one more frame)."""
        return any(not r.text_open or r.closed or r.n_text >= r.emitted for r in self.running.values())

    def _advance(self):
        """One step of the session: ({slot: (request, first new frame, new frames)}, [ids that finished])."""
        # parks: requests of park(rid), then as many waiting live-text requests as the others need slots
        for slot, r in list(self.running.items()):
            if r.paused:
                self._park(slot)
        if self.park_waiting:
            short = sum(self._admissible(r) for r in self.pending) + sum(self._resumable(r) for r in self.parked.values()) \
                - (self.n_slots - len(self.running))
            for slot, r in list(self.running.items()):
                if short <= 0:
                    break
                if self._waiting(r):
                    self._park(slot)
                    short -= 1
        free = [s for s in range(self.n_slots) if s not in self.running]
        for r in [q for q in self.parked.values() if self._resumable(q)][:len(free)]:   # oldest park first
            self._resume(r, free.pop(0))
        batch = []
        for r in [q for q in self.pending if self._admissible(q)][:len(free)]:
            self.pending.remove(r)
            r.slot = free.pop(0)
            batch.append(r)
        if batch:
            args = ([r.slot for r in batch], [r.rid for r in batch], [r.embeds for r in batch], [r.trailing for r in batch])
            kw = {}
            if any(r.sampling is not None for r in batch):
                kw["sampling"] = [r.sampling for r in batch]   # None entries: the session's parameters
            if any(r.voice is not None for r in batch):
                kw["prefixes"] = [r.voice.prefix_id if r.voice is not None else None for r in batch]
            self.eng.admit(*args, **kw)
            for r in batch:
                self.running[r.slot] = r
                if r.voice is not None:
                    r.voice.pending -= 1   # the slot has its own copy of the voice's K/V now
                if r.text_open and not r.closed:
                    self.eng.set_text_open(r.slot, True)
            if self.cstream is not None:
                seeded = [r for r in batch if r.ref_codes is not None]
                banked = [r for r in batch if r.voice is not None and r.voice.bank is not None]
                if len(seeded) + len(banked) < len(batch):
                    self.cstream.reset([r.slot for r in batch if r.ref_codes is None and not any(r is q for q in banked)])
                if seeded:
                    self.cstream.seed([r.slot for r in seeded], [r.ref_codes for r in seeded])
                for bank in sorted({r.voice.bank[0] for r in banked}):   # one copy per bank, no reference decode
                    rs = [r for r in banked if r.voice.bank[0] == bank]
                    self.cstream.copy_from(self.codec.bank_stream(bank), [r.voice.bank[1] for r in rs], [r.slot for r in rs])
                for name in audio.STAGES:   # one reset per stage and setting
                    for args in dict.fromkeys(r.chain[name] for r in batch if name in r.chain):
                        self._stage(name).reset([r.slot for r in batch if r.chain.get(name) == args], *args)
        if not batch and not self._runnable():
            return {}, []   # every running row is open and waiting for text: launch nothing
        n = min([self.packet] + [r.max_frames - r.emitted for r in self.running.values()])
        self.eng.decode(max(n, 1), self.codes)
        torch.cuda.current_stream(self.eng.device).synchronize()
        fd, n_valid, fin = self.eng.progress()
        self.frames_total = fd
        finished, give_up = [], []
        new = {}  # slot -> (request, first new frame, new frames)
        for slot, r in list(self.running.items()):
            have = min(n_valid[slot], r.max_frames)
            new[slot] = (r, r.emitted, have - r.emitted)
            r.emitted = have
            if fin[slot] or have >= r.max_frames:
                self.done[r.rid] = self.codes[slot, :have].to(torch.int64).clone()
                finished.append(r.rid)
                if not fin[slot]:
                    give_up.append(slot)  # horizon reached without EOS: the row is abandoned, its slot is free again
                del self.running[slot]
        if give_up:
            self.eng.release_slots(give_up)
        return new, finished

    def _push_audio(self, new) -> Dict[int, np.ndarray]:
        """One codec step over all slots: slot s takes its new frames codes[s, e0:e0+k] as its count k, idle slots 0.
        Slots of requests with a chain of stages then take their new audio through it (_push_formats), and those whose
        request finished in this step end their clips there (their tails come even without new frames)."""
        if self.cstream is None:
            return {}
        m = max([k for _, _, k in new.values()], default=0)
        ending = [slot for slot, (r, _, _) in new.items() if r.shaped and self.running.get(slot) is not r]
        if m == 0 and not ending:
            return {}
        wav = None
        if m > 0:
            start, counts = [0] * self.n_slots, [0] * self.n_slots
            for slot, (_, e0, k) in new.items():
                start[slot], counts[slot] = e0, k
            idx = (torch.tensor(start)[:, None] + torch.arange(m)[None]).clamp_(max=self.max_frames - 1)
            rows = torch.arange(self.n_slots)[:, None]
            codes = self.codes[rows.to(self.codes.device), idx.to(self.codes.device)].transpose(1, 2)  # [S][G][m]
            wav = self.cstream.push(codes, counts)[:, 0]
        if any(r.shaped for r, _, _ in new.values()):
            return self._push_formats(new, wav, ending)
        wav = wav.cpu().numpy()
        up = self.codec.total_upsample
        return {r.rid: wav[slot, :k * up] for slot, (r, _, k) in new.items() if k > 0}

    def _push_formats(self, new, wav: Optional[torch.Tensor], ending: List[int]) -> Dict[int, np.ndarray]:
        """_push_audio of a step in which some request is shaped, `wav` the codec push's audio on the device (None
        without new frames): the default slots' audio comes back as before, the others' goes through their chains.  One
        launch per stage serves every slot that uses it; a request that finished in the step ends its row in each of
        its stages, and each stage's tail goes on into the next stage's end."""
        up = self.codec.total_upsample
        out: Dict[int, np.ndarray] = {}
        plain = [slot for slot, (r, _, k) in new.items() if not r.shaped and k > 0]
        if plain:
            host = wav[plain].cpu().numpy()
            for i, slot in enumerate(plain):
                out[new[slot][0].rid] = host[i, :new[slot][2] * up]
        x, cnt = wav, {slot: k * up for slot, (r, _, k) in new.items() if r.shaped and k > 0}   # each slot's input
        for name, obj in self.stages.items():
            counts = {slot: c for slot, c in cnt.items() if name in new[slot][0].chain}
            end = [slot for slot in ending if name in new[slot][0].chain]
            if not counts and not end:
                continue
            last = {slot: next(reversed(new[slot][0].chain)) == name for slot in set(counts) | set(end)}
            onward = [slot for slot in sorted(last) if not last[slot]]
            got = obj.push_rows(x if counts else None, counts, end, host=not onward)
            for slot, y in got.items():
                if last[slot] and (y.shape[0] or slot in ending):   # a stage's delay can hold a short push back
                    out[new[slot][0].rid] = y if not onward else y.cpu().numpy()
            cnt = {slot: c for slot, c in cnt.items() if slot not in counts}
            if not onward:
                continue
            cnt.update({slot: int(got[slot].shape[0]) for slot in onward})
            L = max(cnt.values(), default=0)
            nx = torch.zeros(self.n_slots, L, dtype=torch.float32, device=self.eng.device) if L else None
            for slot, c in cnt.items():
                if c:
                    nx[slot, :c] = got[slot] if slot in onward else x[slot, :c]
            x = nx
        return out

    def run(self) -> Dict[int, torch.Tensor]:
        """Drain the queue; returns {request id: (N_i, G) codes}.  Requests with open text must be closed first (or
        be fed through step() / stream() / packets()): run() raises ValueError when nothing pending, running or parked
        can make progress (every running request waits for text, and no other request can take a slot: pending ones
        whose overlay waits for text cannot)."""
        while self.pending or self.running or self.parked:
            if not self._runnable() and not self._can_enter():
                raise ValueError("every request waits for text: close_text() them, or feed them between step()s")
            self.step()
        return self.done

    def _can_enter(self) -> bool:
        """Some pending or resumable parked request can take a slot at the next step: one is free, or will be freed by
        a park."""
        if not (any(self._admissible(r) for r in self.pending) or any(self._resumable(r) for r in self.parked.values())):
            return False
        return len(self.running) < self.n_slots or any(r.paused or (self.park_waiting and self._waiting(r))
                                                       for r in self.running.values())
