"""Live text (SURVEY §8f-2): a row whose next text row has not arrived holds its frame-step instead of reading tts_pad,
so a request whose text arrives piece by piece generates exactly, bit for bit, what it generates with the whole text
given up front — at the engine (holds at frame 0, in mid-launch, across whole launches, beside closed rows), through the
ContinuousBatcher with audio out, with cancelled requests, and at the full 1.7B shape."""
import numpy as np
import pytest
import torch

from oracle import talker as OT
from tests import helpers as Hh
from tests.test_gpu_scheduler_audio import _codec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _sampling(kind, N):
    import qwen3_tts_b200 as q
    if kind == "greedy":
        return q.SamplingParams(do_sample=False, subtalker_dosample=False, max_new_tokens=N + 1, suppress_eos=True, seed=3)
    return q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, subtalker_top_k=50,
                            subtalker_temperature=0.9, repetition_penalty=1.05, max_new_tokens=N + 1, suppress_eos=True, seed=7)


def _tiny_engine(identity=False, max_batch=4):
    """The tiny config, with a code-predictor projection (its input x_cp survives the code-predictor passes) or with
    the Identity one of the 0.6B model (the passes run in place on x_cp, which a held step must put back)."""
    from qwen3_tts_b200.engine import AREngine
    cfg = OT.cfg_tiny()
    cfg.talker.rope_theta = 1e6
    cfg.cp.rope_theta = 1e4
    if identity:
        cfg.cp.hidden_size = cfg.talker.hidden_size
    Wb, _ = Hh.bf16_weights(OT.random_weights(cfg, seed=3))
    return cfg, AREngine(Hh.to_pkg_cfg(cfg), Wb, device=DEV, max_batch=max_batch, max_ctx=160)


def _drive(eng, embs, full, pad, sp, init, opened, launches, N):
    """Static batch prefilled with the first init[b] trailing rows of full[b]; rows in `opened` are open.  `launches`:
    [(frames, {row: rows to append before}, rows to close before)].  After the listed launches every row is closed and
    decoded until it has N frames.  After every launch, progress() must be the committed steps (+1 while held) of a
    host model of the hold rule, and the codes reported so far a prefix of the up-front run.  Returns the hold log."""
    B, G = len(embs), eng.cfg.num_code_groups
    ref = [c.cpu().numpy() for c in eng.generate(embs, full, pad, sp)]
    assert all(r.shape == (N, G) for r in ref)
    cap = max(int(t.shape[0]) for t in full)
    eng.prefill(embs, [t[:n] for t, n in zip(full, init)], pad, sp, trailing_capacity=cap)
    for b in opened:
        eng.set_text_open(b, True)
    codes = torch.zeros(B, 4 * N, G, dtype=torch.int32, device=DEV)
    T, c, is_open = list(init), [0] * B, [b in opened for b in range(B)]
    log = []
    drain = [(8, {}, list(range(B)))] * 8
    for k, (n, app, close) in enumerate(list(launches) + drain):
        if k >= len(launches):   # drain: append whatever is left, close everything, run until every row has N frames
            if min(c) >= N:
                break
            app = {b: int(full[b].shape[0]) - T[b] for b in range(B)}
        for b, m in app.items():
            m = min(m, int(full[b].shape[0]) - T[b])
            if m > 0:
                eng.append_trailing(b, full[b][T[b]:T[b] + m])
                T[b] += m
        for b in close:
            if is_open[b]:
                eng.set_text_open(b, False)
                is_open[b] = False
        eng.decode(n, codes)
        torch.cuda.synchronize()
        held = [False] * B
        for b in range(B):
            commit = min(n, max(0, T[b] - c[b])) if is_open[b] else n
            held[b] = commit < n
            if held[b]:
                log.append((k, b, c[b] + commit, "start" if commit == 0 else "mid"))
            c[b] += commit
        _, nv, fin = eng.progress()
        want = [c[b] + int(held[b]) for b in range(B)]
        assert nv == want and not any(fin), (k, nv, want)
        got = codes.cpu().numpy()
        for b in range(B):
            m = min(want[b], N)
            assert (got[b, :m] == ref[b][:m]).all(), f"launch {k} row {b}: differs from the up-front run at {np.argwhere(got[b, :m] != ref[b][:m])[0]}"
    return log


@pytest.mark.parametrize("identity", [False, True], ids=["projection", "identity"])
@pytest.mark.parametrize("kind", ["sampled", "greedy"])
def test_engine_live_rows_equal_text_given_up_front(kind, identity):
    cfg, eng = _tiny_engine(identity)
    H, N = cfg.talker.hidden_size, 20
    embs, _, pad = Hh.make_inputs(cfg, [11, 7, 9, 6], [0, 0, 0, 0], seed=17)
    g = torch.Generator().manual_seed(5)
    full = [(torch.randn(n, H, generator=g) * 0.1).bfloat16() for n in (9, 6, 7, 5)]
    sp = _sampling(kind, N)
    launches = [
        (3, {}, []),              # row 0 (no text) holds at frame 0; row 1 runs dry at step 2 in mid-launch; row 2 at 3
        (2, {}, []),              # rows 0, 1, 2 held for a whole launch
        (4, {1: 2}, []),          # row 1 commits two more steps and holds again in mid-launch; row 0 still held
        (3, {0: 3, 2: 1}, []),    # row 0 leaves its frame-0 hold; row 2 commits one step and holds
        (5, {0: 6, 1: 2}, [0, 1]),  # rows 0 and 1 get the end of their text and close; row 2 stays held
        (1, {}, []),
        (6, {2: 3}, [2]),
    ]
    # row 3 is never opened: it reads its whole text and then tts_pad beside the held rows
    log = _drive(eng, embs, full, pad, sp, [0, 2, 3, 5], [0, 1, 2], launches, N)
    assert (0, 0, 0, "start") in log and (0, 1, 2, "mid") in log and (2, 1, 4, "mid") in log
    assert {k for k, b, _, _ in log if b == 0} >= {0, 1, 2}     # held across several whole launches
    assert not any(b == 3 for _, b, _, _ in log)
    eng.close()


def _solo(eng, pad, sp, emb, trail, key, frames):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cb = ContinuousBatcher(eng, pad, sp, n_slots=1, packet_frames=4)
    cb.submit(emb, trail, key=key, max_frames=frames)
    return cb.run()[key].cpu().numpy()


def test_batcher_live_requests_with_audio():
    """Two live requests fed piece by piece between steps, one admitted while both are held, and a closed one: each
    request's codes equal its solo up-front run and its chunks the one-shot decode of those codes, bit for bit.  A
    step with no runnable row launches nothing and decodes nothing."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng = _tiny_engine()
    H = cfg.talker.hidden_size
    embs, _, pad = Hh.make_inputs(cfg, [11, 7, 9, 6], [0, 0, 0, 0], seed=21)
    g = torch.Generator().manual_seed(9)
    full = [(torch.randn(n, H, generator=g) * 0.1).bfloat16() for n in (8, 6, 5, 3)]
    sp = _sampling("sampled", 24)
    horizons = [18, 14, 12, 10]
    solo = {i: _solo(eng, pad, sp, embs[i], full[i], i, horizons[i]) for i in range(4)}
    dec = _codec()
    cb = ContinuousBatcher(eng, pad, sp, n_slots=3, packet_frames=4, codec=dec)
    pushes = []
    push = cb.cstream.push
    cb.cstream.push = lambda *a, **k: (pushes.append(1), push(*a, **k))[1]
    fed = {0: 0, 1: 0}

    def feed(rid, m, close=False):
        cb.append_text(rid, full[rid][fed[rid]:fed[rid] + m])
        fed[rid] += m
        if close:
            cb.close_text(rid)

    cb.submit(embs[0], full[0][:0], key=0, max_frames=horizons[0], text_open=True)
    cb.submit(embs[1], full[1][:0], key=1, max_frames=horizons[1], text_open=True)
    actions = {
        0: lambda: None,                                  # both held at frame 0: one frame each
        2: lambda: feed(0, 2),                            # request 2 was admitted beside the two held rows
        3: lambda: feed(1, 6, close=True),
        4: lambda: (feed(0, 3), cb.submit(embs[3], full[3], key=3, max_frames=horizons[3])),
        6: lambda: feed(0, 3, close=True),
    }
    audio, order, frames_seen = {}, [], []
    gen = cb.stream()
    for it, (chunks, finished) in enumerate(gen):
        for rid, a in chunks.items():
            audio.setdefault(rid, []).append(a)
        order += finished
        frames_seen.append(cb.frames_total)
        if it == 1:
            # nothing to admit and both rows wait for text: no launch, no codec step, no frames
            assert chunks == {} and frames_seen[1] == frames_seen[0] and len(pushes) == 1
            cb.submit(embs[2], full[2], key=2, max_frames=horizons[2])
        actions.get(it, lambda: None)()
        assert it < 200
    assert sorted(order) == [0, 1, 2, 3]
    for i in range(4):
        codes = cb.done[i].cpu().numpy()
        assert (codes == solo[i]).all(), f"request {i}: codes differ from its solo up-front run"
        got = np.concatenate(audio[i])
        ref = dec.forward(torch.from_numpy(codes).T[None].to(DEV))[0, 0].cpu().numpy()
        assert np.array_equal(got, ref), f"request {i}: streamed audio differs from the solo decode"
    cb.cstream.close()
    dec.close()
    eng.close()


def test_cancel_pending_held_and_running():
    """cancel() of a pending request, a held live request and a running closed one: the request that reuses a freed
    slot and every other request equal their solo runs; cancelled requests get no result."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng = _tiny_engine()
    H = cfg.talker.hidden_size
    embs, _, pad = Hh.make_inputs(cfg, [11, 7, 9, 6, 8], [0] * 5, seed=31)
    g = torch.Generator().manual_seed(13)
    full = [(torch.randn(n, H, generator=g) * 0.1).bfloat16() for n in (5, 4, 6, 3, 4)]
    sp = _sampling("sampled", 16)
    cb = ContinuousBatcher(eng, pad, sp, n_slots=2, packet_frames=4)
    r0 = cb.submit(embs[0], full[0][:1], key=0, max_frames=12, text_open=True)   # held after its first step
    r1 = cb.submit(embs[1], full[1], key=1, max_frames=15)                      # running, closed
    r2 = cb.submit(embs[2], full[2], key=2, max_frames=10)                      # pending, cancelled
    r3 = cb.submit(embs[3], full[3], key=3, max_frames=10)                      # takes a freed slot
    cb.step()
    assert cb.cancel(r2) and r2 not in [r.rid for r in cb.pending]
    cb.step()
    assert cb.cancel(r0)          # held: its text stopped at one row
    cb.step()                     # request 3 enters request 0's slot
    assert cb.cancel(r1)
    r4 = cb.submit(embs[4], full[4], key=4, max_frames=10)
    out = cb.run()
    assert sorted(out) == [r3, r4] and not cb.cancel(r1) and not cb.cancel(99)
    for i in (3, 4):
        ref = _solo(eng, pad, sp, embs[i], full[i], i, 10)
        assert (out[i].cpu().numpy() == ref).all(), f"request {i} differs from its solo run"
    eng.close()


@pytest.mark.parametrize("n_slots", [32, 8])
def test_full_shape_live_rows_equal_text_given_up_front(n_slots):
    """1.7B shapes, seeded random weights, prompts of at least 128 positions (the batch's attention split count is then
    the same in the live and the up-front run: 1 at 32 rows, 2 at 8): live rows with holds equal the up-front run."""
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.engine import AREngine
    cfg = synthetic.cfg_1p7b()
    W = synthetic.random_tts_weights(cfg, device=DEV, seed=0)
    N = 10
    eng = AREngine(cfg, W, device=DEV, max_batch=n_slots, max_ctx=256)
    del W
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(2)
    lens = [128 + (7 * b) % 29 for b in range(n_slots)]
    embs = [(torch.randn(n, H, generator=g) * 0.5).bfloat16() for n in lens]
    full = [(torch.randn(4 + b % 5, H, generator=g) * 0.1).bfloat16() for b in range(n_slots)]
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    opened = [b for b in range(n_slots) if b % 4 != 3]
    init = [b % 3 if b in opened else int(full[b].shape[0]) for b in range(n_slots)]   # closed rows: their whole text
    launches = [(3, {}, []), (2, {b: 1 for b in opened if b % 2 == 0}, []), (4, {b: 2 for b in opened}, [])]
    log = _drive(eng, embs, full, pad, _sampling("sampled", N), init, opened, launches, N)
    assert any(kind == "start" for *_, kind in log) and any(kind == "mid" for *_, kind in log)
    eng.close()


def test_errors():
    """The engine refuses a bad slot, a slot without a running request, and live text beside hidden-state capture;
    the batcher's append_text / close_text raise ValueError for every request they cannot serve."""
    import ctypes
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng = _tiny_engine()
    H = cfg.talker.hidden_size
    embs, trail, pad = Hh.make_inputs(cfg, [6, 7], [2, 2], seed=1)
    sp = _sampling("greedy", 8)
    eng.prefill(embs, trail, pad, sp, trailing_capacity=8)
    for slot in (-1, 2, 99):
        with pytest.raises(RuntimeError, match="out of range"):
            eng.set_text_open(slot, True)
    hid = torch.zeros(2, 16, H, dtype=torch.bfloat16, device=DEV)
    eng.set_text_open(0, True)
    eng.lib.q3_set_hidden_capture(eng.h, ctypes.c_void_p(hid.data_ptr()), 16)
    with pytest.raises(RuntimeError, match="hidden-state capture"):
        eng.set_text_open(1, True)
    codes = torch.zeros(2, 8, cfg.num_code_groups, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="hidden-state capture"):
        eng.decode(2, codes)
    eng.lib.q3_set_hidden_capture(eng.h, None, 0)
    cb = ContinuousBatcher(eng, pad, sp, n_slots=2, packet_frames=4, max_trailing=6)
    live = cb.submit(embs[0], trail[0], key=0, max_frames=4, text_open=True)
    plain = cb.submit(embs[1], trail[1], key=1, max_frames=2)
    with pytest.raises(ValueError, match="max_trailing"):
        cb.append_text(live, torch.zeros(5, H, dtype=torch.bfloat16))
    with pytest.raises(ValueError, match="not submitted with text_open"):
        cb.append_text(plain, torch.zeros(1, H, dtype=torch.bfloat16))
    with pytest.raises(ValueError, match="unknown"):
        cb.close_text(77)
    cb.step()                     # the plain request reached its horizon of 2 frames: slot 1 is free again
    assert 1 not in cb.running
    with pytest.raises(RuntimeError, match="no running request"):
        eng.set_text_open(1, True)
    cb.close_text(live)
    with pytest.raises(ValueError, match="already closed"):
        cb.append_text(live, torch.zeros(1, H, dtype=torch.bfloat16))
    cb.run()
    with pytest.raises(ValueError, match="has finished"):
        cb.close_text(live)
    gone = cb.submit(embs[0], trail[0], key=5, max_frames=4, text_open=True)
    assert cb.cancel(gone)
    with pytest.raises(ValueError, match="was cancelled"):
        cb.append_text(gone, torch.zeros(1, H, dtype=torch.bfloat16))
    eng.close()
