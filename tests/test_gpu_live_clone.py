"""Live text of ICL voice clones: a request whose prompt waits for K = Lc - R target-text rows is admitted once they
have arrived (or its text closed) and then runs as any live request, so it generates and streams exactly, bit for bit,
what the whole request given up front does — through the batcher with audio at the tiny shape (overlay filled before
and exactly at K, closed short, K = 0, unregistered and registered voices, sampled and greedy, beside ordinary
requests), and at the 1.7B shape with 32 and 8 slots for requests admitted mid-session."""
import numpy as np
import pytest
import torch

from tests.test_gpu_live_text import _sampling
from tests.test_gpu_scheduler_audio import _codec
from tests.test_gpu_voice_prefix import _voice_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (reference text, reference frames, target text, pieces of the text: the first given at submit, then one per step,
# then tts_eos and close; registered voice).  The character processor gives R = len(reference text), T = len(text).
REQS = [
    ("abcd", 9, "Hello there, friend.", [3, 4, 6, 7], False),   # K = 6: filled by the second piece, then trailing text
    ("abcd", 9, "Hello!", [2, 4], False),                        # filled exactly at K by the last piece, then tts_eos
    ("abcd", 9, "Hi", [1, 1], False),                            # closed with the overlay 3 rows short
    ("a longer reference", 9, "Go on then.", [2, 9], False),     # K = 0: an ordinary live request
    ("abcd", 9, "Good day to you.", [0, 5, 11], True),           # a registered voice, no text at submit
    ("abcd", 9, "Plain text.", None, False),                     # not live: the whole request up front
]
HORIZONS = [14, 11, 9, 12, 13, 10]


def _model():
    """The tiny model of the registered-voice tests with one text token per ResizeMLP call, so that rows computed from
    pieces of the text are the rows the whole text gives (a GEMM may round a row differently with its row count)."""
    dec = _codec()
    w = _voice_model(dec)
    tp = w.model._tp
    w.model._tp = lambda t: torch.cat([tp(t[:, j:j + 1]) for j in range(t.shape[1])], dim=1) if t.shape[1] else tp(t)  # noqa: E731
    return w, dec


def _stream(cb, todo, each_step=lambda it: None):
    """Run cb.stream(), calling todo.pop(0)() after each of the first steps and each_step(it) after every step;
    returns {request id: concatenated chunks}."""
    audio = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, a in chunks.items():
            audio.setdefault(rid, []).append(a)
        if todo:
            todo.pop(0)()
        each_step(it)
        assert it < 300
    return {k: np.concatenate(v) for k, v in audio.items()}


@pytest.mark.parametrize("kind", ["sampled", "greedy"])
def test_live_clone_requests_equal_their_up_front_runs(kind):
    from qwen3_tts_b200.model import VoiceClonePromptItem
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    w, dec = _model()
    H = w.model.cfg.talker.hidden_size
    g = torch.Generator().manual_seed(12)
    items = [VoiceClonePromptItem(torch.randint(0, 2000, (L, 16), generator=g), (torch.randn(H, generator=g) * 0.3).bfloat16(),
                                  False, True, ref) for ref, L, _, _, _ in REQS]
    voices = {i: w.register_voice(voice_clone_prompt=[items[i]], language="English") for i, r in enumerate(REQS) if r[4]}
    sp = _sampling(kind, 16)
    up_front = []
    for i, (_, _, text, _, _) in enumerate(REQS):
        (req,), pad = w.build_voice_clone_requests(text, language="English", voice_clone_prompt=[items[i]])
        up_front.append(req)

    # each request alone, whole up front
    solo_codes, solo_audio = {}, {}
    for i, (emb, tr, ref) in enumerate(up_front):
        cb = ContinuousBatcher(w.model.engine, pad, sp, n_slots=1, packet_frames=4, codec=dec)
        cb.submit(emb, tr, key=i, max_frames=HORIZONS[i], ref_codes=ref)
        solo_audio[i] = _stream(cb, [])[i]
        solo_codes[i] = cb.done[i]
        cb.cstream.close()

    # live requests fed piece by piece between steps, beside the up-front one, three slots, admitted at different steps
    cb = ContinuousBatcher(w.model.engine, pad, sp, n_slots=3, packet_frames=4, codec=dec)
    feeds = {}    # request id -> text pieces still to come

    def submit(i):
        ref_text, _, text, pieces, registered = REQS[i]
        if pieces is None:
            emb, tr, ref = up_front[i]
            cb.submit(emb, tr, key=i, max_frames=HORIZONS[i], ref_codes=ref)
            return
        cuts = np.cumsum([0] + pieces).tolist()
        assert cuts[-1] == len(text)
        first = text[:cuts[1]]
        if registered:
            emb, tr, _, ov = w.build_live_clone_request(first, voice=voices[i])
            cb.submit(emb, tr, key=i, max_frames=HORIZONS[i], voice=voices[i], text_open=True, overlay=ov)
        else:
            emb, tr, _, ov = w.build_live_clone_request(first, voice_clone_prompt=items[i], language="English")
            cb.submit(emb, tr, key=i, max_frames=HORIZONS[i], ref_codes=items[i].ref_code, text_open=True, overlay=ov)
        feeds[i] = [text[a:b] for a, b in zip(cuts[1:], cuts[2:])]

    def feed(it):
        for rid in list(feeds):
            if feeds[rid]:
                cb.append_text(rid, w.live_text_rows(feeds[rid].pop(0)))
            else:
                cb.append_text(rid, w.live_text_end())
                cb.close_text(rid)
                del feeds[rid]

    for i in (0, 5, 2):
        submit(i)
    got = _stream(cb, [lambda: submit(1), lambda: submit(4), lambda: submit(3)], feed)
    assert sorted(cb.done) == list(range(len(REQS)))
    for i in range(len(REQS)):
        assert torch.equal(cb.done[i], solo_codes[i]), f"request {i}: codes differ from its up-front run"
        assert np.array_equal(got[i], solo_audio[i]), f"request {i}: streamed audio differs from its up-front run"
    cb.cstream.close()
    for v in voices.values():
        v.close()
    w.model.engine.close()
    dec.close()


@pytest.mark.parametrize("n_slots", [32, 8])
def test_full_shape_live_clones_admitted_mid_session(n_slots):
    """1.7B shapes, seeded random weights, prompts of at least 128 positions (the attention split count is then the same
    in both sessions).  Half the slots run ordinary requests; the other half's requests are live ICL clones whose
    overlay of 15 rows (a 38-frame reference, a 24-token reference text) fills two steps later, admitted then, held for
    text, then closed.  The same session with those requests submitted whole at the step they fill gives the same codes."""
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.engine import AREngine
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg = synthetic.cfg_1p7b()
    W = synthetic.random_tts_weights(cfg, device=DEV, seed=0)
    eng = AREngine(cfg, W, device=DEV, max_batch=n_slots, max_ctx=256)
    del W
    H, K, N = cfg.talker.hidden_size, 15, 10
    g = torch.Generator().manual_seed(6)
    rows = lambda n, s=0.5: (torch.randn(n, H, generator=g) * s).bfloat16().to(DEV)  # noqa: E731
    pad = rows(1, 0.1)[0]
    plain = list(range(n_slots // 2))
    icl = list(range(n_slots // 2, n_slots))
    prompts = {i: rows(128 + (7 * i) % 23 - (K if i in icl else 0)) for i in range(n_slots)}   # known rows
    overlays = {i: rows(K) for i in icl}
    texts = {i: rows(K + 3 + i % 4, 0.1) for i in range(n_slots)}    # the text rows, tts_eos last
    sp = _sampling("sampled", N)

    def session(live):
        cb = ContinuousBatcher(eng, pad, sp, n_slots=n_slots, packet_frames=4)
        for i in plain:
            cb.submit(prompts[i], texts[i], key=i, max_frames=N)
        if live:
            for i in icl:
                cb.submit(prompts[i], texts[i][:2], key=i, max_frames=N, text_open=True, overlay=overlays[i])
        cb.step()
        cb.step()
        assert len(cb.running) == len(plain)
        for i in icl:
            if live:
                cb.append_text(i, texts[i][2:K + 1])   # the overlay is full, one trailing row
            else:
                whole = torch.cat([prompts[i], overlays[i] + texts[i][:K]], 0)
                cb.submit(whole, texts[i][K:], key=i, max_frames=N)
        cb.step()
        assert not cb.pending
        cb.step()
        if live:
            for i in icl:
                cb.append_text(i, texts[i][K + 1:])
                cb.close_text(i)
        return cb.run()

    live, whole = session(True), session(False)
    assert sorted(live) == sorted(whole) == list(range(n_slots))
    for i in range(n_slots):
        assert live[i].shape[0] == N and torch.equal(live[i], whole[i]), f"request {i}: codes differ from the up-front run"
    eng.close()
