"""Voice-clone requests streamed through the continuous batcher and TTSEngine.stream_synthesize: each request's audio is
the part of generate_voice_clone's waveform after the reference (the reference decodes cat(ref_code, codes) and cuts
the reference off, qwen3_tts_model.py:612-631), bit for bit, with ICL and x-vector-only prompts built from raw audio."""
import numpy as np
import pytest
import torch

from tests.test_gpu_e2e import DEV, _proc

pytestmark = pytest.mark.gpu
UP = 1920
KW = dict(max_new_tokens=9, do_sample=True, top_k=50, top_p=1.0, temperature=0.9, repetition_penalty=1.05,
          subtalker_dosample=True, subtalker_top_k=50, subtalker_top_p=1.0, subtalker_temperature=0.9, seed=7)
TEXTS = ["hello there", "second one", "a third text", "four"]


@pytest.fixture(scope="module")
def cloned(tmp_path_factory):
    """Tiny Base checkpoint, prompts from raw audio (ICL with references of 5 and 21 frames, x-vector only), and
    generate_voice_clone's waveforms for TEXTS."""
    from tests.helpers import write_tiny_checkpoint
    from qwen3_tts_b200.model import Qwen3TTSModel
    d = str(tmp_path_factory.mktemp("base"))
    write_tiny_checkpoint(d, device=DEV, seed=0, model_type="base", spk_enc_dim=256)
    m = Qwen3TTSModel.from_pretrained(d, device_map=DEV, processor=_proc, max_batch=8, max_ctx=256, codec_max_frames=128)
    g = np.random.default_rng(1)
    short = (np.clip(g.standard_normal(9000).astype(np.float32) * 0.1, -1, 1), 24000)
    long_ = (np.clip(g.standard_normal(40000).astype(np.float32) * 0.1, -1, 1), 24000)
    items = m.create_voice_clone_prompt([short, short, long_, long_], ref_text=["reference words", None, "longer one", None],
                                        x_vector_only_mode=[False, True, False, True])
    assert [None if it.ref_code is None else it.ref_code.shape[0] for it in items] == [5, None, 21, None]
    wavs, fs = m.generate_voice_clone(TEXTS, language="english", voice_clone_prompt=items, **KW)
    reqs, pad = m.build_voice_clone_requests(TEXTS, language="english", voice_clone_prompt=items)
    yield m, items, wavs, reqs, pad
    m.model.engine.close()


def _session_sp():
    """The parameters generate_voice_clone's call of model.generate samples with."""
    import qwen3_tts_b200 as q
    return q.SamplingParams(min_new_tokens=2, **KW)


def _check(m, i, ref, codes, streamed, want):
    """streamed == decode(cat(ref, codes))[L*UP:] and == the tail of generate_voice_clone's waveform `want`."""
    dec = m.model.speech_tokenizer.decoder
    L = 0 if ref is None else int(ref.shape[0])
    full = codes if ref is None else torch.cat([ref.to(codes.device), codes], 0)
    assert streamed.shape == (codes.shape[0] * UP,), (i, streamed.shape, codes.shape)
    if codes.shape[0]:
        one = dec.forward(full.T[None].to(DEV))[0, 0, L * UP:].cpu().numpy()
        assert np.array_equal(streamed, one), f"request {i}: streamed audio differs from the one-shot decode by {np.abs(streamed - one).max()}"
    assert 0 <= want.shape[0] - streamed.shape[0] <= (1 if L else 0), (i, want.shape, streamed.shape)
    assert np.array_equal(want[want.shape[0] - streamed.shape[0]:], streamed), f"request {i}: differs from generate_voice_clone"


def test_batcher_streams_what_generate_voice_clone_keeps(cloned):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    m, items, wavs, reqs, pad = cloned
    dec = m.model.speech_tokenizer.decoder
    assert [r is None for _, _, r in reqs] == [False, True, False, True]
    cb = ContinuousBatcher(m.model.engine, pad, _session_sp(), n_slots=2, packet_frames=4, codec=dec)
    for i in (0, 1):
        cb.submit(reqs[i][0], reqs[i][1], key=i, ref_codes=reqs[i][2])
    audio = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, a in chunks.items():
            audio.setdefault(rid, []).append(a)
        if it in (0, 2):
            i = 2 if it == 0 else 3
            cb.submit(reqs[i][0], reqs[i][1], key=i, ref_codes=reqs[i][2])
    assert sorted(cb.done) == [0, 1, 2, 3]
    for i, (_, _, ref) in enumerate(reqs):
        got = np.concatenate(audio[i]) if i in audio else np.zeros(0, np.float32)
        _check(m, i, ref, cb.done[i], got, wavs[i])
    with pytest.raises(ValueError, match="codes must lie"):
        cb.submit(reqs[0][0], reqs[0][1], ref_codes=reqs[0][2] + dec.cfg.codebook_size)
    with pytest.raises(ValueError, match="expected an"):
        cb.submit(reqs[0][0], reqs[0][1], ref_codes=reqs[0][2][:, :3])
    with pytest.raises(ValueError, match="frames outside"):
        cb.submit(reqs[0][0], reqs[0][1], ref_codes=torch.zeros(dec.max_frames, dec.cfg.num_quantizers, dtype=torch.long))
    assert not cb.pending
    cb.cstream.close()
    plain = ContinuousBatcher(m.model.engine, pad, _session_sp(), n_slots=2, packet_frames=4)
    with pytest.raises(ValueError, match="codec"):
        plain.submit(reqs[0][0], reqs[0][1], ref_codes=reqs[0][2])


def _tts_engine(m):
    """A TTSEngine over the model's own AR engine and codec decoder."""
    from qwen3_tts_b200.pipeline import TTSEngine
    te = TTSEngine.__new__(TTSEngine)
    te.device, te.ar, te.codec = m.model.device, m.model.engine, m.model.speech_tokenizer.decoder
    te.cfg, te.codec_cfg, te.timing = m.model.cfg, te.codec.cfg, {}
    return te


def test_stream_synthesize_with_reference_codes(cloned):
    m, items, wavs, reqs, pad = cloned
    te = _tts_engine(m)
    dec = te.codec
    embs, trail, refs = [r[0] for r in reqs], [r[1] for r in reqs], [r[2] for r in reqs]
    sp = _session_sp()
    pkts = list(te.stream_synthesize(embs, trail, pad, sp, packet_frames=4, ref_codes=refs))
    got = [np.concatenate([p[b] for p in pkts]) for b in range(len(reqs))]
    codes = [c.to(torch.int64) for c in te.ar.generate(embs, trail, pad, sp)]
    for i in range(len(reqs)):
        _check(m, i, refs[i], codes[i], got[i], wavs[i])
    # the windowed modes: every packet is the forward of its window (reference + generated frames so far)
    for lc in (25, None):
        emitted = [0] * len(reqs)
        for pkt in te.stream_synthesize(embs, trail, pad, sp, packet_frames=4, left_context=lc, ref_codes=refs):
            for b, chunk in enumerate(pkt):
                n = chunk.shape[0] // UP
                if n == 0:
                    continue
                full = codes[b] if refs[b] is None else torch.cat([refs[b].to(DEV), codes[b]], 0)
                end = full.shape[0] - codes[b].shape[0] + emitted[b]
                ctx = end if lc is None else min(lc, end)
                want = dec.forward(full[end - ctx:end + n].T[None].to(DEV))[0, 0, ctx * UP:].cpu().numpy()
                assert np.array_equal(chunk, want), (lc, b, emitted[b])
                emitted[b] += n
        assert emitted == [int(c.shape[0]) for c in codes]
    with pytest.raises(ValueError, match="ref_codes has 1 entries"):
        next(te.stream_synthesize(embs, trail, pad, sp, ref_codes=refs[:1]))
    with pytest.raises(ValueError, match="codes must lie"):
        next(te.stream_synthesize(embs, trail, pad, sp, ref_codes=[refs[0] * 0 - 1] + refs[1:]))
    te._cstream.close()
