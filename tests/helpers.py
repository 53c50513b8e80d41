"""Shared helpers for the parity tests (test infrastructure; may import oracle/)."""
import numpy as np
import torch

from oracle import talker as OT

LOGIT_TOL = 0.06      # |engine - fp32 oracle| on raw logits (logit std ~0.8 with the seeded weights); the
                      # bf16-vs-fp32 gap of the *oracle itself* is ~0.03 (see DESIGN.md §Tolerance)


def to_pkg_cfg(ocfg: OT.TTSCfg):
    import qwen3_tts_b200 as q

    def st(s):
        return q.StackConfig(s.hidden_size, s.num_layers, s.num_heads, s.num_kv_heads, s.head_dim,
                             s.intermediate_size, s.vocab_size, s.rms_eps, s.rope_theta)
    return q.TTSConfig(talker=st(ocfg.talker), cp=st(ocfg.cp), num_code_groups=ocfg.num_code_groups,
                       text_hidden_size=ocfg.text_hidden_size, text_vocab_size=ocfg.text_vocab_size,
                       codec_eos_token_id=ocfg.codec_eos_token_id, codec_pad_id=ocfg.codec_pad_id,
                       codec_bos_id=ocfg.codec_bos_id, tts_bos_token_id=ocfg.tts_bos_token_id,
                       tts_eos_token_id=ocfg.tts_eos_token_id, tts_pad_token_id=ocfg.tts_pad_token_id)


def to_pkg_sampling(sp: OT.SamplingCfg):
    import qwen3_tts_b200 as q
    return q.SamplingParams(**{k: getattr(sp, k) for k in q.SamplingParams.__dataclass_fields__})


def bf16_weights(W):
    """bf16-rounded weights: (bf16 dict for the engine, fp32 upcast of the SAME values for the oracle)."""
    Wb = {k: v.to(torch.bfloat16) for k, v in W.items()}
    Wf = {k: v.to(torch.float32) for k, v in Wb.items()}
    return Wb, Wf


def make_inputs(cfg, lens, trail_lens, seed=0):
    g = torch.Generator().manual_seed(seed)
    H = cfg.talker.hidden_size
    embs = [(torch.randn(l, H, generator=g) * 0.5).bfloat16() for l in lens]
    trail = [(torch.randn(n, H, generator=g) * 0.1).bfloat16() for n in trail_lens]
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    return embs, trail, pad


def run_engine_forced(eng, embs, trail, pad, sp_pkg, forced: np.ndarray, dev):
    """Teacher-forced run with raw-logit capture.  forced: (B, N, G) int."""
    B, N, G = forced.shape
    V, Vc = eng.cfg.talker.vocab_size, eng.cfg.cp.vocab_size
    f = torch.from_numpy(forced.astype(np.int32)).to(dev).contiguous()
    tl = torch.zeros(N + 1, B, V, dtype=torch.float32, device=dev)
    cl = torch.zeros(N, G - 1, B, Vc, dtype=torch.float32, device=dev)
    eng.set_debug(f, N, tl, cl)
    eng.prefill(embs, trail, pad, sp_pkg)
    codes = torch.zeros(B, N, G, dtype=torch.int32, device=dev)
    eng.decode(N, codes)
    torch.cuda.synchronize()
    prog = eng.progress()
    eng.set_debug(None, 0, None, None)
    return codes.cpu().numpy(), tl.cpu().numpy(), cl.cpu().numpy(), prog


# ---------------------------------------------------------------------------------------------- synthetic HF checkpoints
def tiny_checkpoint_configs():
    """config.json dictionaries (reference format: core/models/configuration_qwen3_tts.py,
    core/tokenizer_12hz/configuration_qwen3_tts_tokenizer_v2.py) for a tiny model matching synthetic.cfg_tiny()."""
    talker = dict(vocab_size=3072, hidden_size=256, intermediate_size=512, num_hidden_layers=3, num_attention_heads=4,
                  num_key_value_heads=2, head_dim=128, rms_norm_eps=1e-6, rope_theta=1e6,
                  rope_scaling=dict(mrope_section=[24, 20, 20], interleaved=True, rope_type="default"),
                  num_code_groups=16, text_hidden_size=256, text_vocab_size=1000, codec_eos_token_id=2150,
                  codec_think_id=2154, codec_nothink_id=2155, codec_think_bos_id=2156, codec_think_eos_id=2157,
                  codec_pad_id=2148, codec_bos_id=2149, spk_id={"Alice": 3000, "bob": 3001},
                  spk_is_dialect={"Alice": False, "bob": False}, codec_language_id={"english": 2050, "chinese": 2055},
                  code_predictor_config=dict(vocab_size=2048, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                                             num_attention_heads=4, num_key_value_heads=2, head_dim=128,
                                             rms_norm_eps=1e-6, rope_theta=1e4, num_code_groups=16))
    top = dict(model_type="qwen3_tts", talker_config=talker, speaker_encoder_config={}, tokenizer_type="qwen3_tts_tokenizer_12hz",
               tts_model_size="1b7", tts_model_type="custom_voice", tts_pad_token_id=996, tts_bos_token_id=997,
               tts_eos_token_id=998)
    tok = dict(model_type="qwen3_tts_tokenizer_12hz", encoder_valid_num_quantizers=16, input_sample_rate=24000,
               output_sample_rate=24000, decode_upsample_rate=1920, encode_downsample_rate=1920,
               decoder_config=dict(codebook_size=2048, codebook_dim=64, hidden_size=64, latent_dim=64,
                                   num_attention_heads=4, num_key_value_heads=4, sliding_window=6, intermediate_size=96,
                                   num_hidden_layers=2, num_quantizers=16, upsample_rates=[8, 5, 4, 3],
                                   upsampling_ratios=[2, 2], decoder_dim=256, rms_norm_eps=1e-5, rope_theta=10000),
               encoder_config=dict(model_type="mimi", num_filters=8, hidden_size=64, num_hidden_layers=2,
                                   num_attention_heads=4, num_key_value_heads=4, head_dim=16, intermediate_size=96,
                                   sliding_window=6, codebook_size=64, codebook_dim=32,
                                   vector_quantization_hidden_dimension=32, upsample_groups=64))
    gen = dict(do_sample=True, top_k=40, temperature=0.8, max_new_tokens=64)
    return top, tok, gen


def write_tiny_checkpoint(directory, device="cpu", sharded=False, seed=0, model_type="custom_voice", spk_enc_dim=24):
    """Write a complete synthetic checkpoint directory in the reference's on-disk format; returns what was written
    (tts weights, decoder weights, encoder weights) for comparison."""
    import json
    import os
    from safetensors.torch import save_file
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.config import EncoderConfig
    top, tok, gen = tiny_checkpoint_configs()
    os.makedirs(os.path.join(directory, "speech_tokenizer"), exist_ok=True)
    cfg = synthetic.cfg_tiny()
    W = {k: v.cpu().contiguous() for k, v in synthetic.random_tts_weights(cfg, device=device, seed=seed, with_text=True).items()}
    if model_type == "base":   # Base checkpoints carry the ECAPA speaker encoder (modeling_qwen3_tts.py:1822-1825)
        import dataclasses as _dc
        scfg = _dc.replace(synthetic.cfg_speaker_encoder_tiny(), enc_dim=spk_enc_dim)
        top = dict(top, tts_model_type="base",
                   speaker_encoder_config=dict(mel_dim=scfg.mel_dim, enc_dim=scfg.enc_dim, enc_channels=list(scfg.enc_channels),
                                               enc_kernel_sizes=list(scfg.enc_kernel_sizes), enc_dilations=list(scfg.enc_dilations),
                                               enc_attention_channels=scfg.enc_attention_channels,
                                               enc_res2net_scale=scfg.enc_res2net_scale, enc_se_channels=scfg.enc_se_channels))
        for k, v in synthetic.random_speaker_encoder_weights(scfg, seed=seed + 3).items():
            W["speaker_encoder." + k] = v.to(torch.bfloat16).contiguous()
    else:
        top = dict(top, tts_model_type=model_type)
        W["speaker_encoder.fc.weight"] = torch.zeros(4, 4, 1, dtype=torch.bfloat16)  # must be skipped by the loader
    json.dump(top, open(os.path.join(directory, "config.json"), "w"))
    json.dump(gen, open(os.path.join(directory, "generation_config.json"), "w"))
    if sharded:
        keys = sorted(W)
        half = len(keys) // 2
        parts = {"model-00001-of-00002.safetensors": keys[:half], "model-00002-of-00002.safetensors": keys[half:]}
        for fn, ks in parts.items():
            save_file({k: W[k] for k in ks}, os.path.join(directory, fn))
        json.dump({"metadata": {}, "weight_map": {k: fn for fn, ks in parts.items() for k in ks}},
                  open(os.path.join(directory, "model.safetensors.index.json"), "w"))
    else:
        save_file(W, os.path.join(directory, "model.safetensors"))
    d = tok["decoder_config"]
    ccfg = q.CodecConfig(codebook_size=d["codebook_size"], codebook_dim=d["codebook_dim"], hidden_size=d["hidden_size"],
                         latent_dim=d["latent_dim"], num_heads=4, num_kv_heads=4, head_dim=16, sliding_window=6,
                         intermediate_size=96, num_layers=2, decoder_dim=256)
    DW = {k: v.cpu().float().contiguous() for k, v in synthetic.random_codec_weights(ccfg, device=device, seed=seed).items()}
    ecfg = synthetic.cfg_encoder_tiny()
    EW = {k: v.contiguous() for k, v in synthetic.random_encoder_weights(ecfg, seed=seed + 2).items()}
    sd = {"decoder." + k: v for k, v in DW.items()}
    sd.update({"encoder." + k: v for k, v in EW.items()})
    json.dump(tok, open(os.path.join(directory, "speech_tokenizer", "config.json"), "w"))
    save_file(sd, os.path.join(directory, "speech_tokenizer", "model.safetensors"))
    return cfg, W, ccfg, DW, ecfg, EW


def report_parity(name, record):
    """Parity figures the GPU tests measure (free-running exact-match rates, worst logit errors): printed, and
    collected into the JSON file named by $Q3_PARITY_REPORT when that is set."""
    import json, os
    record = {k: (float(v) if isinstance(v, (np.floating, float)) else int(v) if isinstance(v, (np.integer,)) else v) for k, v in record.items()}
    print(f"[parity] {name}: {json.dumps(record)}")
    path = os.environ.get("Q3_PARITY_REPORT")
    if not path:
        return
    try:
        data = json.load(open(path)) if os.path.exists(path) else {}
        data[name] = record
        json.dump(data, open(path, "w"), indent=1, sort_keys=True)
    except OSError:
        pass
