"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and exports every
symbol include/qwen3tts_b200.h declares (no compute calls without a GPU)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "qwen3tts_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(q3_[a-z0-9_]+)\s*\(", hdr)))


def test_library_builds_and_exports_the_abi_2_header_symbols():
    from qwen3_tts_b200 import _lib, build
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    syms = _declared_symbols()
    assert "q3_decode" in syms and "q3_codec_forward" in syms
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f"symbols declared in the header but not exported: {missing}"
    assert sorted(_lib.AR_SYMBOLS + _lib.CODEC_SYMBOLS) == syms
    lib.q3_abi_version.restype = ctypes.c_int
    assert lib.q3_abi_version() == 2


def test_engine_fails_loudly_without_gpu():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from qwen3_tts_b200 import _lib
    lib = _lib.load()
    cfg = _lib.EngineCfg()
    for s in (cfg.talker, cfg.cp):
        s.hidden_size, s.num_layers, s.num_heads, s.num_kv_heads, s.head_dim = 256, 1, 4, 2, 128
        s.intermediate_size, s.vocab_size, s.rms_eps = 512, 2048, 1e-6
    cfg.num_code_groups, cfg.has_cp_projection, cfg.codec_eos_token_id = 16, 0, 2000
    cfg.max_batch, cfg.max_ctx, cfg.device = 4, 128, 0
    h = ctypes.c_void_p()
    rc = lib.q3_engine_create(ctypes.byref(cfg), ctypes.byref(h))
    assert rc != 0 and b"CUDA" in lib.q3_last_error()
    # the codec encoder and the Python wrappers refuse a CPU device as well (no fallback anywhere)
    ec = _lib.CodecEncCfg()
    ec.n_ratios, ec.head_dim, ec.num_heads, ec.hidden_size = 1, 16, 4, 64
    ec.num_quantizers, ec.num_semantic_quantizers, ec.codebook_dim, ec.max_frames = 16, 1, 32, 16
    rc = lib.q3_codec_enc_create(ctypes.byref(ec), ctypes.byref(h))
    assert rc != 0 and b"CUDA" in lib.q3_last_error()
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.codec_encoder import CodecEncoder
    with pytest.raises(RuntimeError):
        CodecEncoder(synthetic.cfg_encoder_tiny(), {}, device="cpu")


def test_sass_is_sm90a_with_wgmma_tma():
    """The shipped cubins target sm_90a; the codec/prefill GEMM carries wgmma (HGMMA) fed by TMA tile loads
    (UTMALDG); the frame-step kernel stages its weights with bulk TMA copies into shared memory (UBLKCP.S.G) completed on mbarriers (SYNCS...TRYWAIT), prefetches KV rows with cp.async (LDGSTS) and runs the
    batch-in-N mma.sync (HMMA)."""
    import subprocess
    from qwen3_tts_b200 import build
    path = build.build()
    out = subprocess.run(["cuobjdump", "-lelf", path], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "UBLKCP.S.G", "SYNCS.PHASECHK.TRANS64.TRYWAIT", "LDGSTS", "HMMA"):
        assert mnemonic in sass, f"{mnemonic} missing from SASS"
