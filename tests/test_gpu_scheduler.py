"""Continuous batching (SURVEY §8f-4): a request admitted into a RUNNING batch generates exactly what it generates
alone, and what the static batch of the reference's call shape generates for the same Philox row key."""
import numpy as np
import pytest
import torch

from oracle import talker as OT
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _setup():
    from qwen3_tts_b200.engine import AREngine
    cfg = OT.cfg_tiny()
    cfg.talker.rope_theta = 1e6
    cfg.cp.rope_theta = 1e4
    Wb, _ = Hh.bf16_weights(OT.random_weights(cfg, seed=3))
    eng = AREngine(Hh.to_pkg_cfg(cfg), Wb, device=DEV, max_batch=4, max_ctx=160)
    lens = [6, 9, 7, 11, 5]
    embs, trail, pad = Hh.make_inputs(cfg, lens, [2, 0, 3, 1, 0], seed=17)
    return cfg, eng, embs, trail, pad


def test_admitted_row_equals_alone_and_static():
    import qwen3_tts_b200 as q
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng, embs, trail, pad = _setup()
    sp = q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, subtalker_top_k=50,
                          subtalker_temperature=0.9, repetition_penalty=1.05, max_new_tokens=13, suppress_eos=True, seed=5)
    horizons = [12, 5, 12, 7, 9]
    # ---- every request alone (a one-slot session; the Philox row key is the request id)
    alone = {}
    for i in range(len(embs)):
        cb = ContinuousBatcher(eng, pad, sp, n_slots=1, packet_frames=4)
        cb.submit(embs[i], trail[i], key=i, max_frames=horizons[i])
        alone[i] = cb.run()[i].cpu().numpy()
        assert alone[i].shape == (horizons[i], cfg.num_code_groups)
    # ---- all five through two slots: rows 2, 3, 4 are admitted while another row is in mid-utterance
    cb = ContinuousBatcher(eng, pad, sp, n_slots=2, packet_frames=4)
    for i in range(len(embs)):
        cb.submit(embs[i], trail[i], key=i, max_frames=horizons[i])
    order = []
    while cb.pending or cb.running:
        order += cb.step()
    out = cb.done
    assert sorted(order) == list(range(len(embs))) and order[0] == 1  # the short request left first, its slot was reused
    for i in range(len(embs)):
        got = out[i].cpu().numpy()
        assert got.shape == alone[i].shape, (i, got.shape)
        assert (got == alone[i]).all(), f"request {i} differs from its solo run at {np.argwhere(got != alone[i])[0]}"
    # ---- the static batch (reference call shape): rows 0 and 1 carry the Philox keys 0 and 1
    st = eng.generate(embs[:2], trail[:2], pad, sp)
    for i in range(2):
        ref = st[i].cpu().numpy()[:horizons[i]]
        assert (ref == alone[i]).all(), f"static row {i} differs from the session run"
    eng.close()


def _alone(eng, pad, sp, emb, trail, key, frames):
    """What one request generates alone: a one-slot session whose Philox row key is `key`."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cb = ContinuousBatcher(eng, pad, sp, n_slots=1, packet_frames=4)
    cb.submit(emb, trail, key=key, max_frames=frames)
    return cb.run()[key].cpu().numpy()


def test_rejected_admission_changes_nothing():
    """An admission that fails on its second row changes no row: its first row (a prompt of max_ctx - 1 positions,
    which would overflow the KV cache at the next decode) is not admitted, the running request and a later valid
    admission generate what each generates alone."""
    import qwen3_tts_b200 as q
    cfg, eng, embs, trail, pad = _setup()
    sp = q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, subtalker_top_k=50,
                          subtalker_temperature=0.9, repetition_penalty=1.05, max_new_tokens=25, suppress_eos=True, seed=5)
    G, H, max_trailing = cfg.num_code_groups, cfg.talker.hidden_size, 4
    g = torch.Generator().manual_seed(23)
    long = (torch.randn(eng.max_ctx - 1, H, generator=g) * 0.5).bfloat16()
    empty = torch.zeros(0, H, dtype=torch.bfloat16)
    too_long = (torch.randn(max_trailing + 1, H, generator=g) * 0.1).bfloat16()
    eng.session_begin(4, pad, sp, max_trailing=max_trailing)
    codes = torch.zeros(4, 32, G, dtype=torch.int32, device=DEV)
    eng.admit([3], [0], [embs[0]], [trail[0]])
    eng.decode(4, codes)
    rejected = [  # (slots, prompts, trailing texts, error)
        ([0, 0, 1], [long, embs[1], embs[2]], [trail[0], trail[1], trail[2]], "slot 0 admitted twice"),
        ([0, 1, 2], [long, empty, embs[2]], [trail[0], trail[1], trail[2]], "prompt length 0 out of range"),
        ([0, 1, 2], [long, embs[1], embs[2]], [trail[0], too_long, trail[2]], f"trailing length {max_trailing + 1} exceeds"),
    ]
    for slots, prompts, trails, err in rejected:
        with pytest.raises(RuntimeError, match=err):
            eng.admit(slots, [10, 11, 12], prompts, trails)
        eng.decode(4, codes)   # no progress() in between: it would clear a stale `active` flag of row 0
    eng.admit([1], [1], [embs[1]], [trail[1]])
    eng.decode(8, codes)
    torch.cuda.synchronize()
    got = codes.cpu().numpy()
    for slot, key, frames in ((3, 0, 24), (1, 1, 8)):
        ref = _alone(eng, pad, sp, embs[key], trail[key], key, frames)
        assert (got[slot, :frames] == ref).all(), f"request {key} differs from its solo run at {np.argwhere(got[slot, :frames] != ref)[0]}"
    eng.close()


def test_rejected_prefill_changes_nothing():
    """A static batch of another size rejected for its second row leaves the running batch's decode bit-identical."""
    import dataclasses
    import qwen3_tts_b200 as q
    cfg, eng, embs, trail, pad = _setup()
    sp = q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, max_new_tokens=9,
                          suppress_eos=True, seed=5)
    G, H = cfg.num_code_groups, cfg.talker.hidden_size
    ref = torch.zeros(2, 8, G, dtype=torch.int32, device=DEV)
    eng.prefill(embs[:2], trail[:2], pad, sp)
    eng.decode(8, ref)
    codes = torch.zeros(2, 8, G, dtype=torch.int32, device=DEV)
    eng.prefill(embs[:2], trail[:2], pad, sp)
    eng.decode(4, codes)
    with pytest.raises(RuntimeError, match="prompt length 0 out of range"):
        eng.prefill([embs[2], torch.zeros(0, H, dtype=torch.bfloat16), embs[3]], trail[2:5], pad,
                    dataclasses.replace(sp, seed=99))
    eng.decode(4, codes)
    torch.cuda.synchronize()
    assert (codes.cpu().numpy() == ref.cpu().numpy()).all()
    eng.close()


def test_eos_frees_the_slot_and_trims():
    """Rows that sample EOS leave the session at their own frame; their codes are trimmed like :2283-2290."""
    import qwen3_tts_b200 as q
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, eng, embs, trail, pad = _setup()
    sp = q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=0, temperature=3.0, subtalker_top_k=50,
                          repetition_penalty=1.0, max_new_tokens=41, suppress_eos=False, seed=11)
    cb = ContinuousBatcher(eng, pad, sp, n_slots=3, packet_frames=4)
    for i in range(len(embs)):
        cb.submit(embs[i], trail[i], key=100 + i)
    out = cb.run()
    assert sorted(out) == [100 + i for i in range(len(embs))]
    for rid, c in out.items():
        c = c.cpu().numpy()
        assert c.shape[1] == cfg.num_code_groups and 0 <= c.shape[0] <= 40
        assert (c[:, 0] != cfg.codec_eos_token_id).all()  # the EOS frame itself is dropped
    eng.close()


def test_streaming_text_input_equals_text_given_up_front():
    """trailing_text_hidden rows appended while the row is generating (before the frame that consumes them) give the
    same codes as the whole text at prefill (modeling_qwen3_tts.py:1689-1692: frame t adds trailing[t], then tts_pad)."""
    import qwen3_tts_b200 as q
    cfg, eng, embs, trail, pad = _setup()
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(3)
    trail = [(torch.randn(7, H, generator=g) * 0.1).bfloat16(), (torch.randn(5, H, generator=g) * 0.1).bfloat16()]
    sp = q.SamplingParams(do_sample=True, max_new_tokens=11, suppress_eos=True, seed=9)
    ref = [c.cpu().numpy() for c in eng.generate(embs[:2], trail, pad, sp)]
    eng.prefill(embs[:2], [t[:2] for t in trail], pad, sp, trailing_capacity=16)
    codes = torch.zeros(2, 10, cfg.num_code_groups, dtype=torch.int32, device=DEV)
    eng.decode(2, codes)                      # frames 0 and 1 consume the two rows given at prefill
    eng.append_trailing(0, trail[0][2:4])
    eng.append_trailing(1, trail[1][2:])
    eng.decode(2, codes)
    eng.append_trailing(0, trail[0][4:])
    eng.decode(6, codes)
    torch.cuda.synchronize()
    got = codes.cpu().numpy()
    for b in range(2):
        assert (got[b] == ref[b]).all(), f"row {b} differs at {np.argwhere(got[b] != ref[b])[0]}"
    eng.close()
