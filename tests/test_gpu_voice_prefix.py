"""Registered voices: a request admitted with a prefix's K/V copied into its slot and only its own rows prefilled
generates exactly, bit for bit, what the admission of cat(prefix rows, own rows) generates — at the engine (tiny shape,
projection and Identity code predictors, greedy and sampled; 1.7B shape at 32 and 8 slots, where the suffix-only and
the full admissions pick different prefill tile widths), across the prefix lifecycle, and through the batcher with
audio, where an ICL voice's codec row is copied from the reference bank instead of decoding the reference."""
import numpy as np
import pytest
import torch

from tests import helpers as Hh
from tests.test_gpu_live_text import _sampling, _tiny_engine
from tests.test_gpu_scheduler_audio import _codec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rows(g, n, H, scale=0.5):
    return (torch.randn(n, H, generator=g) * scale).bfloat16()


def _session(eng, pad, sp, n_slots, admissions, N):
    """Admissions [(frames to decode before, slots, keys, embeds, trailing, prefixes or None)]; then decode until N
    frames.  Returns the codes of every slot and the rows' frame counts."""
    G = eng.cfg.num_code_groups
    eng.session_begin(n_slots, pad, sp, max_trailing=8)
    codes = torch.zeros(n_slots, 2 * N, G, dtype=torch.int32, device=DEV)
    for before, slots, keys, embs, trails, prefixes in admissions:
        if before:
            eng.decode(before, codes)
        kw = {} if prefixes is None else {"prefixes": prefixes}
        eng.admit(slots, keys, embs, trails, **kw)
    eng.decode(N, codes)
    torch.cuda.synchronize()
    _, nv, _ = eng.progress()
    return codes.cpu().numpy(), nv


def _check_twin(eng, pad, sp, n_slots, admissions, prefix_rows, N):
    """The admissions with prefixes, then the same session admitting cat(prefix rows, own rows): equal codes."""
    got, nv = _session(eng, pad, sp, n_slots, admissions, N)
    full = [(b, s, k, [e if p is None else torch.cat([prefix_rows[p], e], 0) for e, p in zip(es, ps or [None] * len(es))], t, None)
            for b, s, k, es, t, ps in admissions]
    want, nv2 = _session(eng, pad, sp, n_slots, full, N)
    assert nv == nv2
    for b in range(n_slots):
        assert np.array_equal(got[b, :nv[b]], want[b, :nv[b]]), f"slot {b}: codes differ from the full admission"
    return got, nv


@pytest.mark.parametrize("identity", [False, True])
@pytest.mark.parametrize("kind", ["greedy", "sampled"])
def test_engine_prefixed_admission_equals_full_admission(kind, identity):
    cfg, eng = _tiny_engine(identity, max_batch=6)
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(11)
    pad = _rows(g, 1, H, 0.1)[0]
    rows = {}
    for n in (9, 14):
        p = _rows(g, n, H)
        rows[eng.create_prefix(p)] = p
    pa, pb = list(rows)
    s = [_rows(g, n, H) for n in (3, 5, 1, 11, 4, 7)]
    t = [_rows(g, n, H, 0.1) for n in (2, 0, 4, 3, 1, 5)]
    N = 10
    adm = [(0, [0, 1, 2, 3], [0, 1, 2, 3], s[:4], t[:4], [pa, pa, pb, None]),
           (3, [4, 5], [4, 5], s[4:], t[4:], [pb, None])]
    _, nv = _check_twin(eng, pad, _sampling(kind, 2 * N), 6, adm, rows, N)
    assert min(nv) >= N - 3
    eng.close()


@pytest.mark.parametrize("n_slots", [32, 8])
def test_full_shape_prefixed_admission_equals_full_admission(n_slots):
    """1.7B shapes, seeded random weights, full prompts of 128 rows or more; the prefill GEMMs of the suffix-only
    admission run over M = sum of suffix rows, those of the full admission over M = sum of prompt rows."""
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.engine import AREngine
    cfg = synthetic.cfg_1p7b()
    W = synthetic.random_tts_weights(cfg, device=DEV, seed=0)
    eng = AREngine(cfg, W, device=DEV, max_batch=n_slots, max_ctx=256)
    del W
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(4)
    pad = _rows(g, 1, H, 0.1)[0]
    rows = {}
    for n in (120, 126):
        p = _rows(g, n, H)
        rows[eng.create_prefix(p)] = p
    ids = list(rows)
    pre = [ids[b % 2] for b in range(n_slots)]
    suf = [_rows(g, 8 + (5 * b) % 17, H) for b in range(n_slots)]
    tr = [_rows(g, 2 + b % 4, H, 0.1) for b in range(n_slots)]
    assert min(rows[p].shape[0] + s.shape[0] for p, s in zip(pre, suf)) >= 128
    # gemm_pick_bn (csrc/gemm_sm90.cu): 128-wide tiles once the M x N tiles fill every SM, else 64
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    pick = lambda N, M: 128 if N > 64 and -(-M // 128) * -(-N // 128) >= sms else 64  # noqa: E731
    t = cfg.talker
    m_suffix = sum(s.shape[0] for s in suf)
    m_full = m_suffix + sum(rows[p].shape[0] for p in pre)
    gemms = {"qkv": (t.num_heads + 2 * t.num_kv_heads) * t.head_dim, "o": H, "gate_up": 2 * t.intermediate_size, "down": H}
    differ = [k for k, N in gemms.items() if pick(N, m_suffix) != pick(N, m_full)]
    assert differ, "the suffix-only and the full admission pick the same tile widths"
    _check_twin(eng, pad, _sampling("sampled", 9), n_slots, [(0, list(range(n_slots)), list(range(n_slots)), suf, tr, pre)],
                rows, 8)
    eng.close()


def test_prefix_lifecycle():
    """Creating and freeing prefixes between decodes leaves running rows' codes unchanged; a freed id is refused and
    has no length; prefixes survive session_begin; an admission with P + S >= max_ctx, an empty suffix or a bad id on
    one request admits no row and leaves the running rows as they were."""
    cfg, eng = _tiny_engine(max_batch=4)
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(5)
    pad = _rows(g, 1, H, 0.1)[0]
    sp = _sampling("sampled", 24)
    pa_rows, pb_rows = _rows(g, 8, H), _rows(g, 6, H)
    pa, pb = eng.create_prefix(pa_rows), eng.create_prefix(pb_rows)
    assert eng.prefix_length(pa) == 8 and eng.prefix_length(pb) == 6
    s = [_rows(g, n, H) for n in (4, 3, 2)]
    t = [_rows(g, n, H, 0.1) for n in (2, 3, 1)]
    G = cfg.num_code_groups

    def run(disturb):
        eng.session_begin(4, pad, sp, max_trailing=8)
        codes = torch.zeros(4, 24, G, dtype=torch.int32, device=DEV)
        eng.admit([0, 1], [0, 1], s[:2], t[:2], prefixes=[pa, None])
        eng.decode(3, codes)
        if disturb:
            pc = eng.create_prefix(_rows(g, 5, H))
            eng.decode(2, codes)
            eng.free_prefix(pc)
            assert eng.prefix_length(pc) == -1
            max_ctx = eng.max_ctx
            long_id = eng.create_prefix(_rows(g, max_ctx - 3, H))
            for bad_prefix, bad_rows, why in ((long_id, s[2][:1].repeat(3, 1), "out of range"),
                                              (pb, s[2][:0], "out of range"), (pc, s[2], "does not exist"),
                                              (-7, s[2], "does not exist")):
                with pytest.raises(RuntimeError, match=f"request 1: .*{why}"):
                    eng.admit([2, 3], [2, 3], [s[2], bad_rows], [t[2], t[2]], prefixes=[pb, bad_prefix])
            eng.free_prefix(long_id)
            with pytest.raises(RuntimeError, match="does not exist"):
                eng.free_prefix(long_id)
            eng.decode(3, codes)
        else:   # the same launches
            eng.decode(2, codes)
            eng.decode(3, codes)
        eng.admit([2], [2], [s[2]], [t[2]], prefixes=[pb])
        eng.decode(8, codes)
        torch.cuda.synchronize()
        return codes.cpu().numpy(), eng.progress()[1]

    quiet, nv = run(False)
    busy, nv2 = run(True)
    assert nv == nv2 and nv[:3] == [16, 16, 8]
    for b in range(3):
        assert np.array_equal(quiet[b, :nv[b]], busy[b, :nv[b]]), f"slot {b}: codes changed by the prefix calls"
    with pytest.raises(RuntimeError, match="out of range"):
        eng.create_prefix(_rows(g, 0, H))
    with pytest.raises(RuntimeError, match="out of range"):
        eng.create_prefix(_rows(g, eng.max_ctx - 1, H))
    eng.close()


def _voice_model(dec):
    """A tiny Qwen3TTSModel on the GPU with the character processor of the CPU voice tests and `dec` as its codec."""
    from types import SimpleNamespace
    from oracle import talker as OT
    from qwen3_tts_b200.model import Qwen3TTSForConditionalGenerationB200 as M, Qwen3TTSModel
    from tests.test_voice_prefix_cpu import _processor
    cfg = OT.cfg_tiny()
    cfg.talker.rope_theta, cfg.cp.rope_theta = 1e6, 1e4
    W = {k: v.to(torch.bfloat16) for k, v in OT.random_weights(cfg, seed=6, with_text=True, text_vocab=1000).items()}
    m = M(Hh.to_pkg_cfg(cfg), W, device=DEV, spk_id={"alice": 3000}, spk_is_dialect={"alice": False},
          codec_language_id={"english": 2050}, tts_model_type="base", max_batch=4, max_ctx=256)
    m.speech_tokenizer = SimpleNamespace(decoder=dec)
    return Qwen3TTSModel(m, _processor)


def test_batcher_voices_stream_what_unregistered_requests_stream():
    """Voices of every kind (custom voice, voice design, x-vector clone, ICL clones with 5- and 21-frame references,
    both layouts) and a live request of a non-ICL voice: each request's streamed chunks equal, bit for bit, those of the
    same request submitted unregistered (prefix rows + its rows, and ref_codes), and no admission of a registered ICL
    voice decodes its reference."""
    from qwen3_tts_b200.model import VoiceClonePromptItem
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    dec = _codec()
    w = _voice_model(dec)
    H = w.model.cfg.talker.hidden_size
    g = torch.Generator().manual_seed(8)
    voices = []
    w.model.tts_model_type = "custom_voice"
    voices.append(w.register_voice(speaker="alice", language="English"))
    w.model.tts_model_type = "voice_design"
    voices.append(w.register_voice(instruct="Calm and low.", non_streaming_mode=True))
    w.model.tts_model_type = "base"
    xv = VoiceClonePromptItem(None, (torch.randn(H, generator=g) * 0.3).bfloat16(), True, False)
    voices.append(w.register_voice(voice_clone_prompt=xv, language="English"))
    for L, ref_text, nsm in ((5, "a reference text", False), (21, "short", True), (21, "ref", False)):
        it = VoiceClonePromptItem(torch.randint(0, 2000, (L, 16), generator=g), (torch.randn(H, generator=g) * 0.3).bfloat16(),
                                  False, True, ref_text)
        voices.append(w.register_voice(voice_clone_prompt=it, language="English", non_streaming_mode=nsm))
    texts = ["Hello there.", "Good day to you.", "One two three.", "Voice cloning.", "Hi.", "Another text."]
    reqs = [w.build_voice_request(txt, v) for txt, v in zip(texts, voices)]
    pad = reqs[0][2]
    sp = _sampling("sampled", 24)
    horizons = [12, 10, 14, 9, 11, 8, 13]
    live_v = voices[0]
    live_suf, live_tr, _ = w.build_voice_request("Hi", live_v, live=True)
    later = torch.cat([w.live_text_rows(" all."), w.live_text_end()], 0)

    def run(registered):
        cb = ContinuousBatcher(w.model.engine, pad, sp, n_slots=3, packet_frames=4, codec=dec)
        seeds = []
        seed = cb.cstream.seed
        cb.cstream.seed = lambda rows, codes: (seeds.append(list(rows)), seed(rows, codes))[1]
        todo = []
        for i, (v, (suf, tr, _)) in enumerate(zip(voices, reqs)):
            if registered:
                todo.append(lambda i=i, v=v, suf=suf, tr=tr: cb.submit(suf, tr, key=i, max_frames=horizons[i], voice=v))
            else:
                todo.append(lambda i=i, v=v, suf=suf, tr=tr: cb.submit(torch.cat([v.prefix, suf], 0), tr, key=i,
                                                                       max_frames=horizons[i], ref_codes=v.ref_codes))
        if registered:   # the live request: its first token up front, the rest appended while it runs
            todo.append(lambda: cb.submit(live_suf, live_tr, key=6, max_frames=horizons[6], voice=live_v, text_open=True))
        else:            # the same rows given up front
            todo.append(lambda: cb.submit(torch.cat([live_v.prefix, live_suf], 0), torch.cat([live_tr, later], 0), key=6,
                                          max_frames=horizons[6]))
        for f in todo[:3]:
            f()
        todo = todo[3:]
        audio = {}
        for it, (chunks, _) in enumerate(cb.stream()):
            for rid, a in chunks.items():
                audio.setdefault(rid, []).append(a)
            if todo:
                todo.pop(0)()
            if registered and 6 in [r.rid for r in cb.running.values()] and it % 2 == 0:
                r = next(r for r in cb.running.values() if r.rid == 6)
                if not r.closed:
                    cb.append_text(6, later)
                    cb.close_text(6)
            assert it < 300
        cb.cstream.close()
        return {k: np.concatenate(v) for k, v in audio.items()}, seeds, cb.done

    got, seeds, done = run(True)
    want, _, want_done = run(False)
    assert seeds == [], f"a registered ICL voice's admission decoded its reference: {seeds}"
    assert sorted(got) == sorted(want) == list(range(7))
    for k in range(7):
        assert torch.equal(done[k], want_done[k]), f"request {k}: codes differ from the unregistered request"
        assert np.array_equal(got[k], want[k]), f"request {k}: streamed audio differs from the unregistered request"
    for v in voices:
        v.close()
    w.model.engine.close()
    dec.close()
