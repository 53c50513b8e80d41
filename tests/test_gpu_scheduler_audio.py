"""Audio out of the continuous batcher: every request's concatenated stream() chunks equal the one-shot codec forward
of its codes alone bit for bit, while requests enter and leave the session's slots at different frames."""
import numpy as np
import pytest
import torch

from tests.test_gpu_scheduler import _setup

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _codec():
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.codec import CodecDecoder
    ccfg = q.CodecConfig(codebook_size=2048, codebook_dim=64, hidden_size=64, latent_dim=64, num_heads=4, num_kv_heads=4,
                         head_dim=16, sliding_window=6, intermediate_size=96, num_layers=2, decoder_dim=256)
    return CodecDecoder(ccfg, synthetic.random_codec_weights(ccfg, device="cpu", seed=0), device=DEV, max_frames=64)


def test_stream_chunks_equal_solo_decode_of_each_request():
    """Five requests through two slots, admitted at different steps (three are submitted while the session runs).
    The talker's EOS row is scaled up so that rows sample EOS once min_new_tokens allows it; horizons 2 and 3 end
    before that, so at least one request leaves at its horizon and the others may leave at EOS."""
    import qwen3_tts_b200 as q
    from qwen3_tts_b200.engine import AREngine
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    from oracle import talker as OT
    from tests import helpers as Hh
    cfg, eng, embs, trail, pad = _setup()
    eng.close()
    W = OT.random_weights(cfg, seed=3)
    W["talker.codec_head.weight"][cfg.codec_eos_token_id] *= 30.0
    Wb, _ = Hh.bf16_weights(W)
    eng = AREngine(Hh.to_pkg_cfg(cfg), Wb, device=DEV, max_batch=4, max_ctx=160)
    dec = _codec()
    sp = q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, subtalker_top_k=50,
                          subtalker_temperature=0.9, repetition_penalty=1.05, max_new_tokens=21, suppress_eos=False,
                          min_new_tokens=4, seed=5)
    horizons = [20, 3, 20, 2, 16]
    alone = {}
    for i in range(len(embs)):
        cb = ContinuousBatcher(eng, pad, sp, n_slots=1, packet_frames=4)
        cb.submit(embs[i], trail[i], key=i, max_frames=horizons[i])
        alone[i] = cb.run()[i].cpu().numpy()
    lens = [alone[i].shape[0] for i in range(len(embs))]
    assert any(n < h for n, h in zip(lens, horizons)), f"no request sampled EOS: {lens}"
    assert any(n == h for n, h in zip(lens, horizons))
    cb = ContinuousBatcher(eng, pad, sp, n_slots=2, packet_frames=4, codec=dec)
    for i in (0, 1):
        cb.submit(embs[i], trail[i], key=i, max_frames=horizons[i])
    audio, order = {}, []
    for it, (chunks, finished) in enumerate(cb.stream()):
        for rid, a in chunks.items():
            assert a.dtype == np.float32 and a.shape[0] % 1920 == 0 and a.shape[0] > 0
            audio.setdefault(rid, []).append(a)
        order += finished
        if it == 0:
            cb.submit(embs[2], trail[2], key=2, max_frames=horizons[2])
            cb.submit(embs[3], trail[3], key=3, max_frames=horizons[3])
        if it == 2:
            cb.submit(embs[4], trail[4], key=4, max_frames=horizons[4])
    assert sorted(order) == list(range(len(embs)))
    for i in range(len(embs)):
        codes = cb.done[i].cpu().numpy()
        assert (codes == alone[i]).all(), f"request {i}: codes differ from its solo run"
        got = np.concatenate(audio[i]) if i in audio else np.zeros(0, np.float32)
        assert got.shape == (codes.shape[0] * 1920,), (i, got.shape, codes.shape)
        if codes.shape[0]:
            ref = dec.forward(torch.from_numpy(codes).T[None].to(DEV))[0, 0].cpu().numpy()
            assert np.array_equal(got, ref), f"request {i}: streamed audio differs from the solo decode by {np.abs(got - ref).max()}"
    cb.cstream.close()
    dec.close()
    eng.close()
