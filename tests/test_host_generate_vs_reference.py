"""Row a1 (composite generate(): prefill assembly) — our PyTorch host code against the reference's own
`Qwen3TTSForConditionalGeneration.generate`, whose call into `talker.generate` (seam B) was intercepted by
oracle/make_golden.py (`reference`): the kwargs it received are recorded in tests/golden/reference_checks.* (the
embedding rows as a fixed sample of 16 hidden columns)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import talker as OT

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
Z = np.load(os.path.join(GOLD, "reference_checks.npz"))
META = json.load(open(os.path.join(GOLD, "reference_checks.json")))


def _setup():
    from tests import helpers as Hh
    cfg = OT.cfg_tiny()
    cfg.talker.rope_theta, cfg.cp.rope_theta = 1e6, 1e4
    W = OT.random_weights(cfg, seed=2, with_text=True, text_vocab=1000)
    spk_id = {"alice": 3000, "bob": 3001}
    lang = {"english": 2050, "chinese": 2055, "sichuan_dialect": 2060}
    dial = {"alice": False, "bob": "sichuan_dialect"}
    from qwen3_tts_b200.model import Qwen3TTSForConditionalGenerationB200
    ours = Qwen3TTSForConditionalGenerationB200.__new__(Qwen3TTSForConditionalGenerationB200)
    Qwen3TTSForConditionalGenerationB200.__init__(ours, Hh.to_pkg_cfg(cfg), W, device="cpu", spk_id=spk_id, spk_is_dialect=dial,
                                                  codec_language_id=lang, engine=object())
    ours.dtype = torch.float32
    # float32 copies of the exact same weights for an exact comparison
    g = lambda k: W[k].float()  # noqa: E731
    ours.text_embedding = g("talker.model.text_embedding.weight")
    ours.fc1_w, ours.fc1_b = g("talker.text_projection.linear_fc1.weight"), g("talker.text_projection.linear_fc1.bias")
    ours.fc2_w, ours.fc2_b = g("talker.text_projection.linear_fc2.weight"), g("talker.text_projection.linear_fc2.bias")
    ours.codec_embedding = g("talker.model.codec_embedding.weight")
    ours.cp_embeddings = [g(f"talker.code_predictor.model.codec_embedding.{j}.weight") for j in range(15)]
    return cfg, ours


def _ids(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 990, (1, n), generator=g)


def _ref_kwargs(name):
    """the recorded talker.generate kwargs; embeddings restricted to the recorded hidden columns"""
    return {"inputs_embeds": torch.from_numpy(Z[name + "_embeds"]), "attention_mask": torch.from_numpy(Z[name + "_mask"]).long(),
            "trailing_text_hidden": torch.from_numpy(Z[name + "_trailing"]), "tts_pad_embed": torch.from_numpy(Z[name + "_pad"])}


def _check(ref_kw, embeds, trailing, pad):
    cols = torch.from_numpy(Z["gen_cols"])
    assert torch.allclose(ref_kw["tts_pad_embed"].reshape(-1), pad, atol=1e-6)
    embeds, trailing, pad = [e[:, cols] for e in embeds], [t[:, cols] for t in trailing], pad[cols]
    x, mask = ref_kw["inputs_embeds"], ref_kw["attention_mask"]
    B, L, _ = x.shape
    assert B == len(embeds)
    for b in range(B):
        n = int(mask[b].sum())
        assert embeds[b].shape[0] == n
        assert torch.allclose(x[b, L - n:], embeds[b], atol=1e-6), b
        assert float(x[b, :L - n].abs().max()) == 0.0 if n < L else True
    tr = ref_kw["trailing_text_hidden"]
    for b in range(B):
        t = trailing[b]
        assert torch.allclose(tr[b, :t.shape[0]], t, atol=1e-6)
        if t.shape[0] < tr.shape[1]:
            assert torch.allclose(tr[b, t.shape[0]:], pad.expand(tr.shape[1] - t.shape[0], -1), atol=1e-6)


@pytest.mark.parametrize("non_streaming", [True, False])
def test_custom_voice_and_voice_design_prefill(non_streaming):
    cfg, ours = _setup()
    input_ids = [_ids(3 + T + 5, 10 + T) for T in (6, 11, 4)]
    instruct_ids = [None, _ids(9, 50), _ids(5, 51)]
    langs = ["english", "auto", "chinese"]
    spks = ["alice", "bob", None]
    name = "gen_custom_" + ("ns" if non_streaming else "s")
    kw = META[name + "_talker_kwargs"]
    e, t, pad = ours.build_prefill(input_ids, instruct_ids, None, None, langs, spks, non_streaming)
    _check(_ref_kwargs(name), e, t, pad)
    # talker kwargs the engine must honour (:2044-2066)
    assert kw["min_new_tokens"] == 2 and kw["eos_token_id"] == cfg.codec_eos_token_id
    V = cfg.talker.vocab_size
    assert kw["suppress_tokens"] == [i for i in range(V - 1024, V) if i != cfg.codec_eos_token_id]
    if non_streaming:
        assert [x.shape[0] for x in e] == [3 + 6 + (6 + 1) + 1, 9 + 3 + 6 + (11 + 1) + 1, 5 + 3 + 5 + 0 + (4 + 1) + 1]  # row 1: dialect speaker => language tag present


@pytest.mark.parametrize("non_streaming", [True, False])
def test_voice_clone_icl_and_xvector_prefill(non_streaming):
    cfg, ours = _setup()
    g = torch.Generator().manual_seed(3)
    input_ids = [_ids(3 + 7 + 5, 20), _ids(3 + 30 + 5, 21), _ids(3 + 5 + 5, 22)]
    ref_ids = [_ids(3 + 6 + 2, 30), _ids(3 + 4 + 2, 31), None]
    H = cfg.talker.hidden_size
    vcp = dict(ref_code=[torch.randint(0, 2000, (9, 16), generator=g), torch.randint(0, 2000, (5, 16), generator=g), None],
               ref_spk_embedding=[torch.randn(H, generator=g) for _ in range(3)],
               x_vector_only_mode=[False, False, True], icl_mode=[True, True, False])
    langs = ["english", "chinese", "auto"]
    e, t, pad = ours.build_prefill(input_ids, None, ref_ids, vcp, langs, None, non_streaming)
    _check(_ref_kwargs("gen_clone_" + ("ns" if non_streaming else "s")), e, t, pad)


def test_unknown_speaker_and_language_raise():
    _, ours = _setup()
    with pytest.raises(NotImplementedError):
        ours.build_prefill([_ids(12, 1)], None, None, None, ["english"], ["carol"], True)
    with pytest.raises(NotImplementedError):
        ours.build_prefill([_ids(12, 1)], None, None, None, ["klingon"], ["alice"], True)
