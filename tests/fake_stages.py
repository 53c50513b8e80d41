"""Stand-ins for the row stages of qwen3_tts_b200.audio (TimeStretch, Limiter, Resampler) in CPU batcher tests.

A fake counts like the stage it replaces, through that stage's own count functions, and its output sample j of a clip
is a pattern of j, so a row that lost its state would restart its pattern.  It records every call."""
import numpy as np
import torch

from qwen3_tts_b200 import audio

TS, LIM = audio.TimeStretch, audio.Limiter
DTYPE = {"f32": np.float32, "s16": np.int16, "ulaw": np.uint8}


class FakeStage:
    """reset(rows, *args) gives each row the setting setting(*args); after n inputs a row has emitted emitted(s, n)
    outputs, and a whole clip gives total(s, n); output j is pattern(s, j).  Device outputs are tensors.  `log` holds
    every call, `made` every instance of the class."""
    made: list

    def __init__(self, device, rows, max_in):
        self.rows, self.max_in, self.log = rows, max_in, []
        self.state = [None] * rows    # (setting, inputs so far)
        self.made.append(self)

    def reset(self, rows, *args):
        self.log.append(("reset", list(rows), *args))
        for r in rows:
            self.state[r] = (self.setting(*args), 0)

    def push_rows(self, x, counts, end=(), host=True):
        self.log.append(("push", dict(counts), list(end), host))
        out = {}
        for r in sorted(set(counts) | set(end)):
            s, n = self.state[r]
            n1 = n + counts.get(r, 0)
            y = self.pattern(s, np.arange(self.emitted(s, n), self.total(s, n1) if r in end else self.emitted(s, n1)))
            out[r] = y if host else torch.from_numpy(y)
            self.state[r] = (s, 0 if r in end else n1)
        return out

    def save(self, rows):
        self.log.append(("save", list(rows)))
        return [self.state[r] for r in rows]

    def load(self, rows, state):
        self.log.append(("load", list(rows)))
        for r, s in zip(rows, state):
            self.state[r] = s


# name -> (setting, emitted, total, pattern)
SPECS = {
    "TimeStretch": (TS.hop, lambda ha, n: TS.emitted(n, ha), lambda ha, n: TS.total(n, ha),
                    lambda ha, j: (1000 + j).astype(np.float32)),
    "Limiter": (lambda volume: volume, lambda v, n: LIM.emitted(n), lambda v, n: LIM.total(n),
                lambda v, j: (5000 + j).astype(np.float32)),
    "Resampler": (lambda in_rate, fmt: (*audio.ratio(in_rate, fmt.sample_rate, pitched=True), fmt.encoding),
                  lambda s, n: audio.emitted(n, s[0], s[1]), lambda s, n: audio.total(n, s[0], s[1]),
                  lambda s, j: (j % 251).astype(DTYPE[s[2]])),
}


def install(monkeypatch):
    """Replace the stage classes of audio by fresh fakes; returns {name: fake class}."""
    fakes = {}
    for name, fns in SPECS.items():
        fakes[name] = type(f"Fake{name}", (FakeStage,), dict(made=[], **{k: staticmethod(f) for k, f in zip(
            ("setting", "emitted", "total", "pattern"), fns)}))
        monkeypatch.setattr(audio, name, fakes[name])
    return fakes
