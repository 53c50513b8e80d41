"""Per-request sampling parameters in continuous batching: every admitted request samples with its own parameters and
seed (q3_admit_with_sampling), so requests with different settings share one session and each generates exactly what
it generates alone in a one-slot session whose default is its parameters; bad parameters are refused whole, before
anything changes."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from oracle import talker as OT, sampler as OS, philox
from tests.test_gpu_ar import ENGINE_SAMPLING
from tests.test_gpu_scheduler import _setup

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAX_NEW = 13


def _sp(**kw):
    import qwen3_tts_b200 as q
    return q.SamplingParams(**dict(dict(max_new_tokens=MAX_NEW, suppress_eos=True), **kw))


def _session_default():
    return _sp(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, subtalker_top_k=50,
               subtalker_temperature=0.9, repetition_penalty=1.05, seed=5)


def _requests():
    """Five requests, submission order: the top-p one leaves first and a greedy one takes its slot while the
    temperature-0.7 one is in mid-utterance."""
    return [
        (_sp(top_k=0, top_p=0.8, subtalker_top_k=0, subtalker_top_p=0.8, seed=23), 5),           # generic path
        (_sp(temperature=0.7, top_k=20, subtalker_temperature=0.7, subtalker_top_k=20, seed=22), 12),
        (_sp(do_sample=False, subtalker_dosample=False, seed=21), 12),                           # greedy
        (_sp(repetition_penalty=1.3, min_new_tokens=5, suppress_eos=False, seed=24), 7),
        (_sp(top_k=0, subtalker_top_k=0, seed=25), 9),                                           # full vocabulary
    ]


def _solo(eng, pad, sp, emb, trail, key, horizon, codec=None):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cb = ContinuousBatcher(eng, pad, sp, n_slots=1, packet_frames=4)
    cb.submit(emb, trail, key=key, max_frames=horizon)
    return cb.run()[key].cpu().numpy()


def _first_diff(a, b):
    if a.shape != b.shape:
        return f"shape {a.shape} vs {b.shape}"
    return np.argwhere(a != b)[0].tolist()


def test_mixed_session_equals_each_request_alone():
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng, embs, trail, pad = _setup()
    sp0, reqs = _session_default(), _requests()
    alone = {i: _solo(eng, pad, sp, embs[i], trail[i], i, h) for i, (sp, h) in enumerate(reqs)}
    as_default = {i: _solo(eng, pad, sp0, embs[i], trail[i], i, h) for i, (_, h) in enumerate(reqs)}
    differ = [i for i in alone if alone[i].shape != as_default[i].shape or (alone[i] != as_default[i]).any()]
    assert len(differ) >= 2, f"only requests {differ} differ from the session default: the test would not see the table"
    cb = ContinuousBatcher(eng, pad, sp0, n_slots=2, packet_frames=4)
    for i, (sp, h) in enumerate(reqs):
        cb.submit(embs[i], trail[i], key=i, max_frames=h, sampling=sp)
    order, slot_of = [], {}
    while cb.pending or cb.running:
        order += cb.step()
        for s, r in cb.running.items():
            slot_of.setdefault(r.rid, s)
    assert order[0] == 0 and slot_of[2] == slot_of[0]   # the greedy request reused the top-p request's slot
    for i in range(len(reqs)):
        got = cb.done[i].cpu().numpy()
        assert got.shape == alone[i].shape and (got == alone[i]).all(), f"request {i}: {_first_diff(got, alone[i])}"
    # an explicit copy of the session's parameters is the session's parameters
    cb = ContinuousBatcher(eng, pad, sp0, n_slots=2, packet_frames=4)
    cb.submit(embs[0], trail[0], key=0, max_frames=reqs[0][1], sampling=dataclasses.replace(sp0))
    cb.submit(embs[1], trail[1], key=1, max_frames=reqs[1][1])
    out = cb.run()
    for i in (0, 1):
        got = out[i].cpu().numpy()
        assert got.shape == as_default[i].shape and (got == as_default[i]).all(), f"request {i}: {_first_diff(got, as_default[i])}"
    eng.close()


def _oracle_sp(name, seed, N):
    kw = ENGINE_SAMPLING[name]
    do_sample = kw.get("do_sample", True)
    top_k, top_p, T = kw.get("top_k", 50), kw.get("top_p", 1.0), kw.get("temperature", 0.9)
    return OT.SamplingCfg(do_sample=do_sample, subtalker_dosample=do_sample, top_k=top_k, top_p=top_p, temperature=T,
                          subtalker_top_k=top_k, subtalker_top_p=top_p, subtalker_temperature=T,
                          repetition_penalty=kw.get("repetition_penalty", 1.05), min_new_tokens=kw.get("min_new_tokens", 2),
                          max_new_tokens=N + 1, seed=seed)


@pytest.mark.parametrize("names", [("greedy", "p0.8_k0", "k200", "min_new5"),
                                   ("penalty1.3", "k50_T0.02", "p0.8_k50", "k0_T3")])
def test_each_row_samples_with_its_own_parameters_against_the_oracle(names):
    """One session whose rows carry different ENGINE_SAMPLING configurations and seeds: every draw of row b is held
    to the oracle's processing with ROW b's parameters and philox.uniform(row b's seed, its key, frame, group), by the
    rule of tests/test_gpu_sampler.py."""
    from tests.test_gpu_sampler import sampled_token_error
    from tests import helpers as Hh
    cfg, eng, embs, trail, pad = _setup()
    B, N, G = len(names), 12, cfg.num_code_groups
    keys = [40 + 3 * b for b in range(B)]
    osps = [_oracle_sp(n, 100 + 7 * b + len(n), N) for b, n in enumerate(names)]
    V, Vc = cfg.talker.vocab_size, cfg.cp.vocab_size
    tl = torch.zeros(N + 1, B, V, dtype=torch.float32, device=DEV)
    cl = torch.zeros(N, G - 1, B, Vc, dtype=torch.float32, device=DEV)
    eng.set_debug(None, 0, tl, cl)
    eng.session_begin(B, pad, _sp(seed=77, max_new_tokens=N + 1, suppress_eos=False), max_trailing=8)
    eng.admit(list(range(B)), keys, embs[:B], trail[:B], sampling=[Hh.to_pkg_sampling(s) for s in osps])
    codes = torch.zeros(B, N + 1, G, dtype=torch.int32, device=DEV)
    eng.decode(N, codes)
    torch.cuda.synchronize()
    fd, n_valid, fin = eng.progress()
    eng.set_debug(None, 0, None, None)
    codes, tl, cl = codes.cpu().numpy(), tl.cpu().numpy(), cl.cpu().numpy()
    checked = 0
    for b, (name, sp) in enumerate(zip(names, osps)):
        lp = OT.talker_logits_processors(cfg, sp)

        def check(raw, proc, u, got, what):
            s = proc(raw, sp.top_p)
            if not sp.do_sample:
                assert got == int(np.argmax(s)), (what, got, int(np.argmax(s)))
                return
            err = sampled_token_error(s, proc(raw, 1.0) if sp.top_p < 1.0 else None, sp.top_p, u, got)
            assert err is None, (what, err)

        gen = []
        for f in range(min(fd, N)):
            got = int(codes[b, f, 0])
            check(tl[f, b], lambda x, p: OS.process_logits(x, generated_ids=gen, **dict(lp, top_p=p)),
                  philox.uniform(sp.seed, keys[b], f, 0), got, (name, b, f, 0))
            checked += 1
            gen.append(got)
            if got == cfg.codec_eos_token_id:
                break
            for j in range(G - 1):
                check(cl[f, j, b], lambda x, p: OS.process_logits(x, do_sample=sp.do_sample, temperature=sp.temperature,
                                                                  top_k=sp.top_k, top_p=p),
                      philox.uniform(sp.seed, keys[b], f, j + 1), int(codes[b, f, j + 1]), (name, b, f, j + 1))
    assert checked >= B * 2
    eng.close()


BAD = [(dict(do_sample=True, temperature=0.0), "temperature"), (dict(top_p=1.5), "top_p"),
       (dict(repetition_penalty=math.nan), "repetition_penalty"), (dict(top_k=-1), "top_k")]


def test_bad_parameters_are_refused_whole_and_change_nothing():
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng, embs, trail, pad = _setup()
    sp0, reqs = _session_default(), _requests()
    alone = {i: _solo(eng, pad, reqs[i][0], embs[i], trail[i], i, reqs[i][1]) for i in (0, 1, 2)}
    # ---- an admission whose request 1 of 3 is bad fails whole; nothing is admitted
    cb = ContinuousBatcher(eng, pad, sp0, n_slots=3, packet_frames=4)
    for kw, field in BAD:
        sampling = [reqs[0][0], dataclasses.replace(reqs[1][0], **kw), None]
        with pytest.raises(RuntimeError) as ei:
            eng.admit([0, 1, 2], [0, 1, 2], embs[:3], trail[:3], sampling=sampling)
        msg = str(ei.value)
        assert "request 1:" in msg and f" {field} " in msg, msg
        _, _, fin = eng.progress()
        assert fin == [1, 1, 1], f"a slot was admitted by a failed call: {fin}"
    # ---- the following valid admission generates what each request generates alone
    for i in (0, 1, 2):
        cb.submit(embs[i], trail[i], key=i, max_frames=reqs[i][1], sampling=reqs[i][0])
    out = cb.run()
    for i in (0, 1, 2):
        got = out[i].cpu().numpy()
        assert got.shape == alone[i].shape and (got == alone[i]).all(), f"request {i}: {_first_diff(got, alone[i])}"
    # ---- submit() refuses bad parameters while a session runs; the running requests finish unchanged
    cb = ContinuousBatcher(eng, pad, sp0, n_slots=2, packet_frames=4)
    for i in (1, 2):
        cb.submit(embs[i], trail[i], key=i, max_frames=reqs[i][1], sampling=reqs[i][0])
    cb.step()
    assert len(cb.running) == 2
    for kw, field in BAD:
        with pytest.raises(ValueError, match=field):
            cb.submit(embs[0], trail[0], key=0, sampling=dataclasses.replace(reqs[0][0], **kw))
    with pytest.raises(ValueError, match="max_new_tokens"):
        cb.submit(embs[0], trail[0], key=0, sampling=dataclasses.replace(reqs[0][0], max_new_tokens=MAX_NEW + 1))
    assert not cb.pending
    out = cb.run()
    assert sorted(out) == [1, 2]
    for i in (1, 2):
        got = out[i].cpu().numpy()
        assert got.shape == alone[i].shape and (got == alone[i]).all(), f"request {i}: {_first_diff(got, alone[i])}"
    eng.close()


def test_mixed_session_audio_equals_one_shot_decode():
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    from tests.test_gpu_scheduler_audio import _codec
    cfg, eng, embs, trail, pad = _setup()
    dec = _codec()
    sp0, reqs = _session_default(), _requests()
    cb = ContinuousBatcher(eng, pad, sp0, n_slots=2, packet_frames=4, codec=dec)
    for i in (0, 1):
        cb.submit(embs[i], trail[i], key=i, max_frames=reqs[i][1], sampling=reqs[i][0])
    audio, order = {}, []
    for it, (chunks, finished) in enumerate(cb.stream()):
        for rid, a in chunks.items():
            audio.setdefault(rid, []).append(a)
        order += finished
        if it == 0:
            for i in (2, 3, 4):
                cb.submit(embs[i], trail[i], key=i, max_frames=reqs[i][1], sampling=reqs[i][0])
    assert sorted(order) == list(range(len(reqs)))
    for i in range(len(reqs)):
        codes = cb.done[i].cpu().numpy()
        got = np.concatenate(audio[i]) if i in audio else np.zeros(0, np.float32)
        assert got.shape == (codes.shape[0] * 1920,), (i, got.shape, codes.shape)
        if codes.shape[0]:
            ref = dec.forward(torch.from_numpy(codes).T[None].to(DEV))[0, 0].cpu().numpy()
            assert np.array_equal(got, ref), f"request {i}: streamed audio differs from the one-shot decode by {np.abs(got - ref).max()}"
    cb.cstream.close()
    dec.close()
    eng.close()
