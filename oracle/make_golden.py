"""Mint golden vectors from the REFERENCE's own modules (through oracle/ref_shims.py) and commit them under
tests/golden/.  Run in the build container only:  python -m oracle.make_golden

The reference ships no fixtures (SURVEY §4); these pin the oracle wherever /root/reference is absent (GPU box).
Shapes are deliberately micro (weights travel inside the .npz)."""
import os

import numpy as np
import torch

from . import codec as OC
from . import mimi_encoder as OM
from . import speaker_encoder as OS
from . import ref_driver as R
from . import talker as OT

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def micro_tts_cfg():
    V = 1200
    return OT.TTSCfg(talker=OT.StackCfg(64, 2, 2, 1, 32, 128, V, rope_theta=1e6),
                     cp=OT.StackCfg(32, 2, 2, 1, 32, 64, 64, rope_theta=1e4), text_hidden_size=64, text_vocab_size=100,
                     codec_eos_token_id=V - 10, codec_pad_id=V - 12, codec_bos_id=V - 11, tts_bos_token_id=97,
                     tts_eos_token_id=98, tts_pad_token_id=96)


def micro_codec_cfg():
    return OC.CodecCfg(codebook_size=32, codebook_dim=16, hidden_size=32, latent_dim=32, num_heads=2, num_kv_heads=2,
                       head_dim=16, sliding_window=4, intermediate_size=48, num_layers=2, num_quantizers=16,
                       upsample_rates=(8, 5, 4, 3), upsampling_ratios=(2, 2), decoder_dim=48)


def make_talker():
    from transformers.cache_utils import DynamicCache
    cfg = micro_tts_cfg()
    W = OT.random_weights(cfg, seed=11, with_text=False)
    m = R.build_reference_talker(cfg, text_vocab=100)
    R.load_weights_into_reference(m, {k: v for k, v in W.items()})
    g = torch.Generator().manual_seed(5)
    H, B, lens, N, G = 64, 2, [4, 7], 4, 16
    embs = [torch.randn(l, H, generator=g) * 0.5 for l in lens]
    trail = [torch.randn(n, H, generator=g) * 0.1 for n in (2, 0)]
    pad = torch.randn(H, generator=g) * 0.1
    codes = torch.randint(0, 64, (B, N, G), generator=g)
    codes[:, :, 0] = torch.randint(0, 150, (B, N), generator=g)
    Lmax = max(lens)
    x = torch.zeros(B, Lmax, H)
    mask = torch.zeros(B, Lmax, dtype=torch.long)
    for i, e in enumerate(embs):
        x[i, Lmax - len(e):] = e
        mask[i, Lmax - len(e):] = 1
    cache = DynamicCache()
    m.rope_deltas = None
    tl, cl = [], []
    with torch.no_grad():
        out = m(inputs_embeds=x, attention_mask=mask, past_key_values=cache, use_cache=True, cache_position=torch.arange(Lmax))
        tl.append(out.logits[:, -1].numpy().copy())
        past_hidden = out.past_hidden
        for step in range(N):
            c0 = codes[:, step, 0]
            cpc = DynamicCache()
            e0 = m.get_input_embeddings()(c0[:, None])
            o = m.code_predictor(inputs_embeds=torch.cat((past_hidden, e0), dim=1), past_key_values=cpc, use_cache=True)
            cl.append(o.logits[:, -1].numpy().copy())
            gs = o.generation_steps
            for j in range(1, G - 1):
                o = m.code_predictor(input_ids=codes[:, step, j:j + 1], past_key_values=cpc, use_cache=True, generation_steps=gs)
                gs = o.generation_steps
                cl.append(o.logits[:, -1].numpy().copy())
            hid = [e0] + [m.code_predictor.get_input_embeddings()[i](codes[:, step, i + 1:i + 2]) for i in range(G - 1)]
            xe = torch.cat(hid, dim=1).sum(1, keepdim=True)
            tr = torch.stack([t[step] if step < t.shape[0] else pad for t in trail])[:, None]
            xe = xe + tr
            mask = torch.cat((mask, torch.ones(B, 1, dtype=torch.long)), dim=1)
            cp = torch.tensor([Lmax + step])
            pos = (cp[0] + m.rope_deltas).view(1, B, 1).expand(3, -1, -1)
            mo = m.model(inputs_embeds=xe, attention_mask=mask, position_ids=pos, past_key_values=cache, use_cache=True, cache_position=cp)
            past_hidden = mo.last_hidden_state[:, -1:]
            tl.append(m.codec_head(mo.last_hidden_state)[:, -1].numpy().copy())
    blob = {f"emb{i}": e.numpy() for i, e in enumerate(embs)}  # (the weights are regenerated from the seed)
    blob.update({f"trail{i}": t.numpy() for i, t in enumerate(trail)})
    blob.update(pad=pad.numpy(), codes=codes.numpy(), talker_logits=np.stack(tl), cp_logits=np.stack(cl))
    np.savez_compressed(os.path.join(OUT, "talker_micro.npz"), **blob)
    print("talker_micro.npz", np.stack(tl).shape, np.stack(cl).shape)


def make_codec():
    cfg = micro_codec_cfg()
    W = OC.random_weights(cfg, seed=13)
    m = R.build_reference_codec_decoder(cfg)
    m.load_state_dict(W, strict=False)
    g = torch.Generator().manual_seed(2)
    codes = torch.randint(0, cfg.codebook_size, (2, 16, 9), generator=g)
    with torch.no_grad():
        wav = m(codes)
        wav_c = m.chunked_decode(codes, chunk_size=4, left_context_size=2)
    blob = {f"W::{k}": v.numpy() for k, v in W.items()}
    blob.update(codes=codes.numpy(), wav=wav.numpy(), wav_chunked=wav_c.numpy())
    np.savez_compressed(os.path.join(OUT, "codec_micro.npz"), **blob)
    print("codec_micro.npz", wav.shape, float(wav.abs().max()))


def micro_encoder_cfg():
    return OM.MimiEncCfg(num_filters=4, hidden_size=32, num_layers=2, num_heads=2, head_dim=16, intermediate_size=48,
                         sliding_window=5, codebook_size=32, codebook_dim=16, num_quantizers=32, valid_num_quantizers=16)


def make_encoder():
    """Golden codes from the third-party encoder the reference wraps: transformers MimiModel (installed 5.5.0; the
    reference pins 4.57.3) driven exactly like Qwen3TTSTokenizerV2Model.encode (…v2.py:977-983)."""
    from transformers import MimiConfig, MimiModel
    cfg = micro_encoder_cfg()
    W = OM.random_weights(cfg, seed=17)
    hf = MimiModel(MimiConfig(**cfg.to_hf_kwargs())).eval()
    missing, unexpected = hf.load_state_dict(W, strict=False)
    assert not unexpected, unexpected
    g = torch.Generator().manual_seed(4)
    wav = (torch.randn(2, 15000, generator=g) * 0.1).clamp(-1, 1)  # 16 transformer frames > window 5, 8 code frames
    with torch.no_grad():
        codes = hf.encode(wav[:, None, :], return_dict=True).audio_codes[:, : cfg.valid_num_quantizers]
    blob = {f"W::{k}": v.numpy() for k, v in W.items()}
    blob.update(wav=wav.numpy(), codes=codes.numpy())
    np.savez_compressed(os.path.join(OUT, "encoder_micro.npz"), **blob)
    print("encoder_micro.npz", tuple(codes.shape))


def make_speaker():
    """Golden x-vectors from the reference's own Qwen3TTSSpeakerEncoder (modeling_qwen3_tts.py:300-393) and log-mels from
    its mel_spectrogram (:396-448; the absent librosa filterbank is supplied by oracle.speaker_encoder)."""
    from . import ref_shims
    ref_shims.install()
    from qwen_tts.core.models import modeling_qwen3_tts as RM
    from qwen_tts.core.models.configuration_qwen3_tts import Qwen3TTSSpeakerEncoderConfig
    cfg = OS.cfg_tiny_spk()
    rc = Qwen3TTSSpeakerEncoderConfig(mel_dim=cfg.mel_dim, enc_dim=cfg.enc_dim, enc_channels=list(cfg.enc_channels),
                                      enc_kernel_sizes=list(cfg.enc_kernel_sizes), enc_dilations=list(cfg.enc_dilations),
                                      enc_attention_channels=cfg.enc_attention_channels,
                                      enc_res2net_scale=cfg.enc_res2net_scale, enc_se_channels=cfg.enc_se_channels)
    m = RM.Qwen3TTSSpeakerEncoder(rc).eval()
    W = OS.random_weights(cfg, seed=19)
    m.load_state_dict(W)
    g = torch.Generator().manual_seed(6)
    wav = (torch.randn(2, 6000, generator=g) * 0.1).clamp(-1, 1)
    RM.librosa_mel_fn = lambda sr, n_fft, n_mels, fmin, fmax: OS.slaney_mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
    mel = RM.mel_spectrogram(wav, n_fft=1024, num_mels=cfg.mel_dim, sampling_rate=24000, hop_size=256, win_size=1024,
                             fmin=0, fmax=12000)
    with torch.no_grad():
        emb = m(mel.transpose(1, 2))
    blob = {f"W::{k}": v.numpy() for k, v in W.items()}
    blob.update(wav=wav.numpy(), mel=mel.numpy(), emb=emb.numpy())
    np.savez_compressed(os.path.join(OUT, "speaker_micro.npz"), **blob)
    print("speaker_micro.npz", tuple(mel.shape), tuple(emb.shape))


def _sig(named_shapes):
    """order-free signature of a parameter list: sha256 over the sorted 'name:shape' lines"""
    import hashlib
    return hashlib.sha256("\n".join(sorted(f"{k}:{tuple(v)}" for k, v in named_shapes)).encode()).hexdigest()


def _cols(n, k, seed):
    return np.sort(np.random.default_rng(seed).choice(n, size=min(n, k), replace=False))


def make_reference_checks():
    """What tests/test_oracle_vs_reference.py, tests/test_host_generate_vs_reference.py and the config tests of
    tests/test_checkpoint_cpu.py compare against, recorded from the reference's own modules with the tests' seeded
    inputs.  Large outputs are kept as a fixed, seeded sample of columns / positions (the full argmax rows stay)."""
    import json
    import types
    from transformers.cache_utils import DynamicCache
    from . import ref_shims
    ref_shims.install()
    from qwen_tts.core.models import modeling_qwen3_tts as RM
    from qwen_tts.core.models.configuration_qwen3_tts import Qwen3TTSConfig, Qwen3TTSSpeakerEncoderConfig
    from qwen_tts.core.tokenizer_12hz.configuration_qwen3_tts_tokenizer_v2 import (Qwen3TTSTokenizerV2Config,
                                                                                   Qwen3TTSTokenizerV2DecoderConfig)
    blob, meta = {}, {}
    # ---- talker + code predictor, teacher-forced on the oracle's greedy codes
    cfg = OT.cfg_tiny()
    cfg.talker.rope_theta, cfg.cp.rope_theta = 1e6, 1e4
    W = OT.random_weights(cfg, seed=1)
    m = R.build_reference_talker(cfg)
    R.load_weights_into_reference(m, W)
    torch.manual_seed(0)
    B, lens, H = 3, [5, 9, 7], cfg.talker.hidden_size
    embs = [torch.randn(l, H) * 0.5 for l in lens]
    trail = [torch.randn(n, H) * 0.1 for n in (2, 1, 4)]
    pad = torch.randn(H) * 0.1
    sp = OT.SamplingCfg(do_sample=False, subtalker_dosample=False, max_new_tokens=6, suppress_eos=True)
    codes = torch.stack(OT.generate(W, cfg, embs, trail, pad, sp).codes)
    Lmax = max(lens)
    x = torch.zeros(B, Lmax, H)
    mask = torch.zeros(B, Lmax, dtype=torch.long)
    for i, e in enumerate(embs):
        x[i, Lmax - len(e):] = e
        mask[i, Lmax - len(e):] = 1
    cache = DynamicCache()
    m.rope_deltas = None
    tl, cl = [], []
    with torch.no_grad():
        out = m(inputs_embeds=x, attention_mask=mask, past_key_values=cache, use_cache=True, cache_position=torch.arange(Lmax))
        tl.append(out.logits[:, -1])
        past_hidden = out.past_hidden
        Tt = max(t.shape[0] for t in trail)
        for step in range(codes.shape[1]):
            cpc = DynamicCache()
            e0 = m.get_input_embeddings()(codes[:, step, 0][:, None])
            o = m.code_predictor(inputs_embeds=torch.cat((past_hidden, e0), dim=1), past_key_values=cpc, use_cache=True)
            cl.append(o.logits[:, -1])
            gs = o.generation_steps
            for j in range(1, cfg.num_code_groups - 1):
                o = m.code_predictor(input_ids=codes[:, step, j:j + 1], past_key_values=cpc, use_cache=True, generation_steps=gs)
                gs = o.generation_steps
                cl.append(o.logits[:, -1])
            hid = [e0] + [m.code_predictor.get_input_embeddings()[i](codes[:, step, i + 1:i + 2]) for i in range(cfg.num_code_groups - 1)]
            xe = torch.cat(hid, dim=1).sum(1, keepdim=True)
            tr = torch.stack([t[step] if step < t.shape[0] else pad for t in trail])[:, None]
            xe = xe + (tr if step < Tt else pad.view(1, 1, H))
            mask = torch.cat((mask, torch.ones(B, 1, dtype=torch.long)), dim=1)
            cp = torch.tensor([Lmax + step])
            pos = (cp[0] + m.rope_deltas).view(1, B, 1).expand(3, -1, -1)
            mo = m.model(inputs_embeds=xe, attention_mask=mask, position_ids=pos, past_key_values=cache, use_cache=True, cache_position=cp)
            past_hidden = mo.last_hidden_state[:, -1:]
            tl.append(m.codec_head(mo.last_hidden_state)[:, -1])
    tl, cl = torch.stack(tl).numpy(), torch.stack(cl).numpy()
    ct, cc = _cols(tl.shape[-1], 64, 1), _cols(cl.shape[-1], 64, 2)
    blob.update(tf_codes=codes.numpy(), tf_talker_cols=ct, tf_talker=tl[..., ct], tf_talker_argmax=tl.argmax(-1),
                tf_cp_cols=cc, tf_cp=cl[..., cc], tf_cp_argmax=cl.argmax(-1))
    # ---- leaf ops
    torch.manual_seed(0)
    x = torch.randn(2, 5, 64)
    n = RM.Qwen3TTSRMSNorm(64, eps=1e-6)
    n.weight.data = torch.randn(64)
    blob.update(leaf_rms=n(x).detach().numpy(), leaf_rms_bf16=n.to(torch.bfloat16)(x.bfloat16()).detach().float().numpy(),
                leaf_rotate_half=RM.rotate_half(x).numpy())
    # ---- codec decoder: tiny (forward + chunked) and the default config (names / shapes / a 3-frame forward)
    for name, ccfg in (("tiny", OC.cfg_tiny_codec()), ("default", OC.CodecCfg())):
        Wc = OC.random_weights(ccfg, seed=3)
        mc = R.build_reference_codec_decoder(ccfg)
        sd = mc.state_dict()
        meta[f"codec_{name}_sig"] = _sig((k, v.shape) for k, v in sd.items() if "rotary_emb" not in k)
        meta[f"codec_{name}_numel"] = int(sum(p.numel() for p in mc.parameters()))
        mc.load_state_dict(Wc, strict=False)
        if name == "tiny":
            g = torch.Generator().manual_seed(5)
            c1 = torch.randint(0, ccfg.codebook_size, (2, 16, 13), generator=g)
            c2 = torch.randint(0, ccfg.codebook_size, (2, 16, 40), generator=g)
            with torch.no_grad():
                w1, w2 = mc(c1).numpy(), mc.chunked_decode(c2, chunk_size=16, left_context_size=5).numpy()
            p1, p2 = _cols(w1.shape[-1], 1024, 3), _cols(w2.shape[-1], 1024, 4)
            blob.update(codec_tiny_shape=np.array(w1.shape), codec_tiny_pos=p1, codec_tiny=w1[..., p1],
                        codec_tiny_absmax=np.float32(np.abs(w1).max()), codec_chunked_pos=p2, codec_chunked=w2[..., p2])
        else:
            torch.manual_seed(0)   # the codes of the test's 3-frame forward
            c = torch.randint(0, ccfg.codebook_size, (1, 16, 3))
            with torch.no_grad():
                blob.update(codec_default_codes=c.numpy(), codec_default=mc(c).numpy())
    # ---- speaker encoder and log-mel front end
    for which in ("tiny", "default"):
        scfg = OS.cfg_tiny_spk() if which == "tiny" else OS.SpkEncCfg()
        rc = Qwen3TTSSpeakerEncoderConfig(mel_dim=scfg.mel_dim, enc_dim=scfg.enc_dim, enc_channels=list(scfg.enc_channels),
                                          enc_kernel_sizes=list(scfg.enc_kernel_sizes), enc_dilations=list(scfg.enc_dilations),
                                          enc_attention_channels=scfg.enc_attention_channels,
                                          enc_res2net_scale=scfg.enc_res2net_scale, enc_se_channels=scfg.enc_se_channels)
        ms = RM.Qwen3TTSSpeakerEncoder(rc).eval()
        meta[f"spk_{which}_sig"] = _sig((k, v.shape) for k, v in ms.state_dict().items())
        ms.load_state_dict(OS.random_weights(scfg, seed=1))
        torch.manual_seed(0)
        mels = torch.randn(2, 57, scfg.mel_dim)
        with torch.no_grad():
            blob[f"spk_{which}_emb"] = ms(mels).numpy()
        RM.librosa_mel_fn = lambda sr, n_fft, n_mels, fmin, fmax: OS.slaney_mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
        y = (torch.randn(2, 9000) * 0.1).clamp(-1, 1)
        blob[f"spk_{which}_mel"] = RM.mel_spectrogram(y, n_fft=1024, num_mels=scfg.mel_dim, sampling_rate=24000, hop_size=256,
                                                      win_size=1024, fmin=0, fmax=12000).numpy()
    # ---- composite generate(): the talker.generate kwargs the reference assembles (prefill rows, trailing text, pad)
    from qwen_tts.core.models.modeling_qwen3_tts import Qwen3TTSForConditionalGeneration as RefTop
    gcfg = OT.cfg_tiny()
    gcfg.talker.rope_theta, gcfg.cp.rope_theta = 1e6, 1e4
    Wg = OT.random_weights(gcfg, seed=2, with_text=True, text_vocab=1000)
    talker = R.build_reference_talker(gcfg, text_vocab=1000)
    R.load_weights_into_reference(talker, Wg)
    tc = talker.config
    tc.spk_id, tc.codec_language_id = {"alice": 3000, "bob": 3001}, {"english": 2050, "chinese": 2055, "sichuan_dialect": 2060}
    tc.spk_is_dialect = {"alice": False, "bob": "sichuan_dialect"}
    fake = types.SimpleNamespace(talker=talker, config=types.SimpleNamespace(
        talker_config=tc, tts_bos_token_id=gcfg.tts_bos_token_id, tts_eos_token_id=gcfg.tts_eos_token_id,
        tts_pad_token_id=gcfg.tts_pad_token_id))
    fake.generate_speaker_prompt = types.MethodType(RefTop.generate_speaker_prompt, fake)
    fake.generate_icl_prompt = types.MethodType(RefTop.generate_icl_prompt, fake)
    got = {}

    def cap(**kw):
        got.update(kw)
        raise StopIteration

    talker.generate = cap
    ref_generate = types.MethodType(getattr(RefTop.generate, "__wrapped__", RefTop.generate), fake)

    def ids(n, seed):
        return torch.randint(0, 990, (1, n), generator=torch.Generator().manual_seed(seed))

    hcols = _cols(gcfg.talker.hidden_size, 16, 5)
    blob["gen_cols"] = hcols
    for ns in (True, False):
        for kind in ("custom", "clone"):
            got.clear()
            try:
                if kind == "custom":
                    ref_generate(input_ids=[ids(3 + T + 5, 10 + T) for T in (6, 11, 4)], instruct_ids=[None, ids(9, 50), ids(5, 51)],
                                 languages=["english", "auto", "chinese"], speakers=["alice", "bob", None],
                                 non_streaming_mode=ns, max_new_tokens=7)
                else:
                    g = torch.Generator().manual_seed(3)
                    H = gcfg.talker.hidden_size
                    vcp = dict(ref_code=[torch.randint(0, 2000, (9, 16), generator=g), torch.randint(0, 2000, (5, 16), generator=g), None],
                               ref_spk_embedding=[torch.randn(H, generator=g) for _ in range(3)],
                               x_vector_only_mode=[False, False, True], icl_mode=[True, True, False])
                    ref_generate(input_ids=[ids(3 + 7 + 5, 20), ids(3 + 30 + 5, 21), ids(3 + 5 + 5, 22)],
                                 ref_ids=[ids(3 + 6 + 2, 30), ids(3 + 4 + 2, 31), None], voice_clone_prompt=vcp,
                                 languages=["english", "chinese", "auto"], non_streaming_mode=ns)
            except (StopIteration, RuntimeError):
                pass
            k = f"gen_{kind}_{'ns' if ns else 's'}"
            blob[k + "_mask"] = got["attention_mask"].numpy().astype(np.int8)
            blob[k + "_embeds"] = got["inputs_embeds"][..., hcols].detach().numpy()
            blob[k + "_trailing"] = got["trailing_text_hidden"][..., hcols].detach().numpy()
            blob[k + "_pad"] = got["tts_pad_embed"].reshape(-1).detach().numpy()
            if kind == "custom":
                meta[k + "_talker_kwargs"] = {n: got[n] for n in ("min_new_tokens", "eos_token_id", "suppress_tokens")}
    # ---- configuration classes
    from tests.helpers import tiny_checkpoint_configs
    top, tok, _ = tiny_checkpoint_configs()
    kw = {k: v for k, v in top.items() if k != "model_type"}
    kw["talker_config"] = dict(kw["talker_config"], pad_token_id=None)
    kw["talker_config"]["code_predictor_config"] = dict(kw["talker_config"]["code_predictor_config"], pad_token_id=None)
    meta["tts_config_to_dict"] = Qwen3TTSConfig(**kw).to_dict()
    d = Qwen3TTSConfig(talker_config=dict(pad_token_id=None, code_predictor_config=dict(pad_token_id=None)))
    meta["tts_config_defaults"] = {"top": d.to_dict(), "talker": d.talker_config.to_dict(),
                                   "code_predictor": d.talker_config.code_predictor_config.to_dict()}
    meta["tokenizer_decoder_defaults"] = Qwen3TTSTokenizerV2DecoderConfig().to_dict()
    meta["tokenizer_defaults"] = Qwen3TTSTokenizerV2Config().to_dict()
    meta["tokenizer_config_to_dict"] = Qwen3TTSTokenizerV2Config(**{k: v for k, v in tok.items() if k != "model_type"}).to_dict()
    np.savez_compressed(os.path.join(OUT, "reference_checks.npz"), **blob)
    with open(os.path.join(OUT, "reference_checks.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True, default=lambda o: o.tolist() if hasattr(o, "tolist") else str(o))
    print("reference_checks.npz", len(blob), "arrays")


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    import sys
    which = sys.argv[1:] or ["talker", "codec", "encoder", "speaker", "reference"]
    if "talker" in which:
        make_talker()
    if "codec" in which:
        make_codec()
    if "encoder" in which:
        make_encoder()
    if "speaker" in which:
        make_speaker()
    if "reference" in which:
        make_reference_checks()
