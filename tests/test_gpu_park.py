"""Parked rows (q3_row_park / q3_row_resume / q3_row_discard): a request that leaves its slot and continues later in
another slot, at a later global frame, generates exactly, bit for bit, the codes it generates never parked — at the
engine (tiny shape with the projection and the Identity code predictor, greedy and sampled; a held live-text row; the
1.7B shape at 32 and 8 slots), through the ContinuousBatcher with audio out, and after every refused call.  The
attention split count, the only cross-row input of a row's arithmetic, is the same in both runs of each comparison
(the tiny shape; the 1.7B shape with prompts of at least 128 positions)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import talker as OT
from tests import helpers as Hh
from tests.test_gpu_scheduler_audio import _codec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _sampling(kind, N, suppress_eos=False):
    """Repetition penalty on (the seen bytes matter) and EOS allowed from frame 12 on (n_gen matters)."""
    import qwen3_tts_b200 as q
    if kind == "greedy":
        return q.SamplingParams(do_sample=False, subtalker_dosample=False, repetition_penalty=1.05, max_new_tokens=N + 1,
                                min_new_tokens=12, suppress_eos=suppress_eos, seed=3)
    return q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, subtalker_top_k=50,
                            subtalker_temperature=0.9, repetition_penalty=1.05, max_new_tokens=N + 1, min_new_tokens=12,
                            suppress_eos=suppress_eos, seed=7)


def _engine(identity=False, max_batch=4, max_ctx=160):
    """The tiny config with its EOS row scaled up (rows sample EOS soon after min_new_tokens allows it), with the
    code-predictor projection or the Identity one of the 0.6B model (x_cp is cp.h)."""
    from qwen3_tts_b200.engine import AREngine
    cfg = OT.cfg_tiny()
    cfg.talker.rope_theta = 1e6
    cfg.cp.rope_theta = 1e4
    if identity:
        cfg.cp.hidden_size = cfg.talker.hidden_size
    W = OT.random_weights(cfg, seed=3)
    W["talker.codec_head.weight"][cfg.codec_eos_token_id] *= 30.0
    Wb, _ = Hh.bf16_weights(W)
    return cfg, AREngine(Hh.to_pkg_cfg(cfg), Wb, device=DEV, max_batch=max_batch, max_ctx=max_ctx)


def _progress(eng):
    torch.cuda.synchronize()
    return eng.progress()


def _finish(eng, codes, slots, N, packet=4):
    """Decode until every request of {request: slot} has N frames or has finished; its codes (at most N frames)."""
    for _ in range(64):
        _, nv, fin = _progress(eng)
        if all(fin[s] or nv[s] >= N for s in slots.values()):
            return {r: codes[s, :min(nv[s], N)].cpu().numpy() for r, s in slots.items()}
        eng.decode(packet, codes)
    raise AssertionError("rows did not finish")


def _twin(eng, S, embs, trails, pad, sp, N, k=3, m=4):
    """Requests 0 (A), 1..n-2 and n-1 (C) in a session of S slots.  The reference runs A in slot 0 throughout and
    admits C into slot S-2 at frame k.  The parked run parks A after k frames, admits C into A's slot, runs m frames,
    resumes A into slot S-1 at that later frame, runs m frames, parks A again, runs 2 frames and resumes it into the
    slot it came from.  Returns (reference codes, parked codes) by request."""
    n, G = len(embs), eng.cfg.num_code_groups
    others, C = list(range(1, n - 1)), n - 1
    assert len(others) <= S - 3
    keys = [100 + 7 * i for i in range(n)]
    first = [0] + others

    def begin():
        eng.session_begin(S, pad, sp, max_trailing=16)
        codes = torch.zeros(S, 4 * N + 32, G, dtype=torch.int32, device=DEV)
        eng.admit(first, [keys[i] for i in first], [embs[i] for i in first], [trails[i] for i in first])
        eng.decode(k, codes)
        return codes

    codes = begin()
    eng.admit([S - 2], [keys[C]], [embs[C]], [trails[C]])
    ref = _finish(eng, codes, {**{i: i for i in first}, C: S - 2}, N)

    codes = begin()
    _, nv, fin = _progress(eng)
    assert not fin[0]
    have = nv[0]
    saved = codes[0, :have].clone()
    rec = eng.park(0)
    eng.admit([0], [keys[C]], [embs[C]], [trails[C]])   # C overwrites slot 0's K/V, seen, x_cp and trailing rows
    eng.decode(m, codes)
    eng.resume(rec, S - 1)
    codes[S - 1, :have] = saved
    _, nv, _ = _progress(eng)
    assert nv[S - 1] == have
    eng.decode(m, codes)
    _, nv, fin = _progress(eng)
    assert not fin[S - 1]
    have = nv[S - 1]
    saved = codes[S - 1, :have].clone()
    rec2 = eng.park(S - 1)
    assert rec2 > rec
    eng.decode(2, codes)
    eng.resume(rec2, S - 1)
    codes[S - 1, :have] = saved
    got = _finish(eng, codes, {**{i: i for i in others}, 0: S - 1, C: 0}, N)
    return ref, got


def _check(ref, got):
    assert sorted(ref) == sorted(got)
    for r in ref:
        assert ref[r].shape == got[r].shape and (ref[r] == got[r]).all(), \
            f"request {r}: parked run differs from the never-parked run ({ref[r].shape} vs {got[r].shape})"


@pytest.mark.parametrize("identity", [False, True], ids=["projection", "identity"])
@pytest.mark.parametrize("kind", ["sampled", "greedy"])
def test_engine_parked_row_equals_never_parked(kind, identity):
    cfg, eng = _engine(identity)
    H, N = cfg.talker.hidden_size, 20
    embs, trails, pad = Hh.make_inputs(cfg, [11, 7, 9], [5, 3, 8], seed=17)
    ref, got = _twin(eng, 4, embs, trails, pad, _sampling(kind, N), N)
    _check(ref, got)
    eng.close()


def test_held_row_parked_and_resumed():
    """A live row the last decode left held is parked, its text arrives while it is parked, and it is resumed into
    another slot: progress reports the same n_valid before the park and after the resume, and its codes equal the run
    with the whole text given up front."""
    cfg, eng = _engine()
    H, N, G = cfg.talker.hidden_size, 20, cfg.num_code_groups
    embs, _, pad = Hh.make_inputs(cfg, [11, 7], [0, 0], seed=23)
    g = torch.Generator().manual_seed(4)
    full = [(torch.randn(n, H, generator=g) * 0.1).bfloat16() for n in (7, 4)]
    sp = _sampling("sampled", N)
    eng.session_begin(4, pad, sp, max_trailing=16)
    codes = torch.zeros(4, 4 * N + 32, G, dtype=torch.int32, device=DEV)
    eng.admit([0, 1], [5, 6], embs, full)
    ref = _finish(eng, codes, {0: 0, 1: 1}, N)

    eng.session_begin(4, pad, sp, max_trailing=16)
    codes = torch.zeros(4, 4 * N + 32, G, dtype=torch.int32, device=DEV)
    eng.admit([0, 1], [5, 6], embs, [full[0][:2], full[1]])
    eng.set_text_open(0, True)
    eng.decode(4, codes)                     # row 0 commits frames 0, 1 and holds at frame 2
    _, nv, _ = _progress(eng)
    assert nv[0] == 3
    saved = codes[0, :3].clone()
    rec = eng.park(0)
    eng.decode(3, codes)
    eng.resume(rec, 2)
    _, nv, fin = _progress(eng)
    assert nv[2] == 3 and not fin[2]
    codes[2, :3] = saved
    eng.append_trailing(2, full[0][2:])
    eng.set_text_open(2, False)
    got = _finish(eng, codes, {0: 2, 1: 1}, N)
    _check(ref, got)
    eng.close()


@pytest.mark.parametrize("n_slots", [32, 8])
def test_full_shape_parked_row_equals_never_parked(n_slots):
    """1.7B shapes, seeded random weights, prompts of at least 128 positions (split count 1 at 32 slots, 2 at 8, in
    both runs)."""
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.engine import AREngine
    cfg = synthetic.cfg_1p7b()
    W = synthetic.random_tts_weights(cfg, device=DEV, seed=0)
    N = 10
    eng = AREngine(cfg, W, device=DEV, max_batch=n_slots, max_ctx=256)
    del W
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(2)
    n = n_slots - 1                      # A, n_slots - 3 others and C
    lens = [128 + (7 * b) % 29 for b in range(n)]
    embs = [(torch.randn(L, H, generator=g) * 0.5).bfloat16() for L in lens]
    trails = [(torch.randn(2 + b % 6, H, generator=g) * 0.1).bfloat16() for b in range(n)]
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    ref, got = _twin(eng, n_slots, embs, trails, pad, _sampling("sampled", N), N)
    _check(ref, got)
    eng.close()


def _schedule():
    """Batcher scenario shared with its host-only rehearsal: requests 1..5 are live and fed one text row every one or
    two steps; request 0 is closed and parked / resumed on request; request 6 is closed, parked on request and
    cancelled while parked."""
    horizons = {0: 14, 1: 14, 2: 12, 3: 16, 4: 10, 5: 13, 6: 12}
    text_len = {0: 6, 1: 7, 2: 5, 3: 8, 4: 6, 5: 7, 6: 4}
    return horizons, text_len


def _drive_batcher(cb, embs, rows, horizons, text_len, max_iters=200):
    """Run the scenario on batcher cb; rows(i, a, b) are text rows a..b of request i.  Returns ({id: chunks},
    (record, bank) of request 6 when it was cancelled)."""
    for i in (6, 0):
        cb.submit(embs[i], rows(i, 0, text_len[i]), key=i, max_frames=horizons[i])
    fed = {}
    for i in range(1, 6):
        cb.submit(embs[i], rows(i, 0, 1), key=i, max_frames=horizons[i], text_open=True)
        fed[i] = 1
    audio, cancelled = {}, None
    gen = cb.stream() if cb.cstream is not None else cb.packets()
    for it, (chunks, _) in enumerate(gen):
        for rid, a in chunks.items():
            audio.setdefault(rid, []).append(a)
        for i in list(fed):
            if it % (1 + i % 2) == 0 and fed[i] < text_len[i]:
                cb.append_text(i, rows(i, fed[i], fed[i] + 1))
                fed[i] += 1
                if fed[i] == text_len[i]:
                    cb.close_text(i)
                    del fed[i]
        if it == 0:
            cb.park(0)
            cb.park(6)
        if it == 5:
            cb.resume(0)
        if 6 in cb.parked and cancelled is None:
            r = cb.parked[6]
            cancelled = (r.record, r.bank)
            assert cb.cancel(6)
        assert it < max_iters
    return audio, cancelled


def _moved_slot(moves):
    """Some request was parked and resumed into a slot other than the one it was parked from."""
    last, moved = {}, False
    for kind, rid, slot in moves:
        if kind == "park":
            last[rid] = slot
        else:
            moved = moved or slot != last[rid]
    return moved


def test_batcher_parks_waiting_requests_with_audio():
    """More live requests than slots, fed a row at a time, with park_waiting: every request's codes equal its run in a
    batcher without parking and its chunks the one-shot decode of those codes, bit for bit; parks happened and some
    request resumed into another slot; a request cancelled while parked freed its record and its bank row."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng = _engine()
    H = cfg.talker.hidden_size
    embs, _, pad = Hh.make_inputs(cfg, [11, 7, 9, 6, 8, 10, 5], [0] * 7, seed=41)
    g = torch.Generator().manual_seed(19)
    horizons, text_len = _schedule()
    full = [(torch.randn(text_len[i], H, generator=g) * 0.1).bfloat16() for i in range(7)]
    sp = _sampling("sampled", 16, suppress_eos=True)
    alone = {}
    for i in range(6):
        cb = ContinuousBatcher(eng, pad, sp, n_slots=1, packet_frames=4)
        cb.submit(embs[i], full[i], key=i, max_frames=horizons[i])
        alone[i] = cb.run()[i].cpu().numpy()
    dec = _codec()
    cb = ContinuousBatcher(eng, pad, sp, n_slots=3, packet_frames=4, codec=dec, park_waiting=True)
    audio, cancelled = _drive_batcher(cb, embs, lambda i, a, b: full[i][a:b], horizons, text_len)
    assert _moved_slot(cb.moves), f"no resume into another slot: {cb.moves}"
    assert sorted(cb.done) == list(range(6)) and 6 not in cb.done
    for i in range(6):
        codes = cb.done[i].cpu().numpy()
        assert codes.shape == alone[i].shape and (codes == alone[i]).all(), f"request {i}: codes differ from its unparked run"
        got = np.concatenate(audio[i])
        ref = dec.forward(torch.from_numpy(codes).T[None].to(DEV))[0, 0].cpu().numpy()
        assert got.dtype == np.float32 and np.array_equal(got, ref), f"request {i}: streamed audio differs from the decode"
    record, (bank, row) = cancelled
    with pytest.raises(RuntimeError, match="does not exist"):
        eng.resume(record, 0)
    assert row not in dec._bank_used[bank] and all(len(u) == 0 for u in dec._bank_used)
    cb.cstream.close()
    dec.close()
    eng.close()


def test_refused_calls_change_nothing():
    """Every refusal raises, names the slot or id, and leaves the running rows as they were: the decode after the
    refused calls equals, bit for bit, the same decode without them."""
    cfg, eng = _engine(max_ctx=160)
    H, G, N = cfg.talker.hidden_size, cfg.num_code_groups, 12
    embs, trails, pad = Hh.make_inputs(cfg, [11, 7, 150], [3, 2, 0], seed=29)
    sp = _sampling("sampled", N)
    # a static batch is not a session
    eng.prefill(embs[:2], trails[:2], pad, sp)
    with pytest.raises(RuntimeError, match="session"):
        eng.park(0)
    # a record whose next position is max_ctx: parked, but refused at resume; then a record of an earlier session
    eng.session_begin(4, pad, sp, max_trailing=8)
    codes = torch.zeros(4, 64, G, dtype=torch.int32, device=DEV)
    eng.admit([0], [1], [embs[2]], [trails[2]])
    eng.decode(10, codes)                      # position 150 + 10 = max_ctx
    full = eng.park(0)
    with pytest.raises(RuntimeError, match=f"record {full}: its next position 160 does not fit max_ctx 160"):
        eng.resume(full, 1)
    eng.discard(full)
    eng.admit([0], [1], [embs[0]], [trails[0]])
    old = eng.park(0)

    def start():
        eng.session_begin(4, pad, sp, max_trailing=8)
        c = torch.zeros(4, 64, G, dtype=torch.int32, device=DEV)
        eng.admit([0, 1], [3, 4], embs[:2], trails[:2])
        eng.decode(3, c)
        return c

    codes = start()
    eng.decode(5, codes)
    ref = _finish(eng, codes, {0: 0, 1: 1}, N)

    codes = start()
    with pytest.raises(RuntimeError, match=f"record {old} belongs to an earlier session"):
        eng.resume(old, 2)
    for slot in (-1, 4, 99):
        with pytest.raises(RuntimeError, match=f"slot {slot} out of range"):
            eng.park(slot)
    with pytest.raises(RuntimeError, match="slot 2 has no running request"):
        eng.park(2)                            # never admitted
    eng.admit([2], [5], [embs[0]], [trails[0]])
    eng.release_slots([2])
    with pytest.raises(RuntimeError, match="slot 2 has no running request"):
        eng.park(2)                            # released
    hid = torch.zeros(4, 16, H, dtype=torch.bfloat16, device=DEV)
    eng.lib.q3_set_hidden_capture(eng.h, ctypes.c_void_p(hid.data_ptr()), 16)
    with pytest.raises(RuntimeError, match="hidden-state capture or teacher forcing"):
        eng.park(0)
    eng.lib.q3_set_hidden_capture(eng.h, None, 0)
    forced = torch.full((4, 4, G), -1, dtype=torch.int32, device=DEV)
    eng.set_debug(forced, 4)
    with pytest.raises(RuntimeError, match="hidden-state capture or teacher forcing"):
        eng.park(0)
    eng.set_debug()
    eng.admit([2], [5], [embs[0]], [trails[0]])
    rec = eng.park(2)
    with pytest.raises(RuntimeError, match="slot 2 has no running request"):
        eng.park(2)                            # already parked
    with pytest.raises(RuntimeError, match="slot 0 is still running"):
        eng.resume(rec, 0)
    with pytest.raises(RuntimeError, match="slot 7 out of range"):
        eng.resume(rec, 7)
    eng.discard(rec)
    for bad in (rec, rec + 1000):              # discarded, never parked
        with pytest.raises(RuntimeError, match=f"record {bad} does not exist"):
            eng.resume(bad, 3)
        with pytest.raises(RuntimeError, match=f"record {bad} does not exist"):
            eng.discard(bad)
    eng.admit([2], [5], [embs[0]], [trails[0]])
    rec = eng.park(2)
    eng.resume(rec, 3)
    with pytest.raises(RuntimeError, match=f"record {rec} does not exist"):
        eng.resume(rec, 2)                     # consumed
    eng.release_slots([3])
    eng.decode(5, codes)
    got = _finish(eng, codes, {0: 0, 1: 1}, N)
    _check(ref, got)
    eng.close()


def test_park_cycles_return_memory():
    """100 park -> resume and 100 park -> discard cycles leave the device's free memory where it was."""
    cfg, eng = _engine()
    G = cfg.num_code_groups
    embs, trails, pad = Hh.make_inputs(cfg, [11, 7], [3, 2], seed=37)
    sp = _sampling("greedy", 40, suppress_eos=True)
    eng.session_begin(4, pad, sp, max_trailing=8)
    codes = torch.zeros(4, 64, G, dtype=torch.int32, device=DEV)
    eng.admit([0, 1], [1, 2], embs, trails)
    eng.decode(2, codes)

    def cycles(n):
        for i in range(n):
            eng.resume(eng.park(0), 2 + i % 2)
            eng.resume(eng.park(2 + i % 2), 0)
            eng.discard(eng.park(1))
            eng.admit([1], [2], [embs[1]], [trails[1]])

    cycles(2)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(DEV)[0]
    cycles(100)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info(DEV)[0] == free0
    eng.decode(2, codes)
    _, nv, fin = _progress(eng)
    assert nv[0] == 4 and not fin[0]
    eng.close()
