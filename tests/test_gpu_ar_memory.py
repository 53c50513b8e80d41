"""Device memory of the AR engine: a session does not keep what it admitted, scratch that grows replaces the old block,
a missing or wrong-sized tensor fails finalize with the store's message, and a failed create leaves nothing behind."""
import pytest
import torch

from oracle import talker as OT
from tests import helpers as Hh
from tests.test_gpu_scratch_growth import MiB, _growth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _tiny():
    cfg = OT.cfg_tiny()
    cfg.talker.rope_theta = 1e6
    cfg.cp.rope_theta = 1e4
    Wb, _ = Hh.bf16_weights(OT.random_weights(cfg, seed=3))
    return cfg, Wb


def _engine(cfg, Wb, max_batch=4, max_ctx=256):
    from qwen3_tts_b200.engine import AREngine
    return AREngine(Hh.to_pkg_cfg(cfg), Wb, device=DEV, max_batch=max_batch, max_ctx=max_ctx)


def _greedy(max_new_tokens=8):
    import qwen3_tts_b200 as q
    return q.SamplingParams(do_sample=False, subtalker_dosample=False, max_new_tokens=max_new_tokens, suppress_eos=True)


def test_admissions_do_not_pile_up():
    """The engine reads an admission's prompt and trailing text only in work queued during the call, so the session
    keeps none of them: admitting into the same slot again and again holds the framework's allocated memory within
    one admission of its level after the first round."""
    cfg, Wb = _tiny()
    eng = _engine(cfg, Wb, max_batch=1, max_ctx=1024)
    H, G = cfg.talker.hidden_size, cfg.num_code_groups
    g = torch.Generator().manual_seed(0)
    prompt = (torch.randn(512, H, generator=g) * 0.5).bfloat16().to(DEV)
    trail = (torch.randn(32, H, generator=g) * 0.1).bfloat16().to(DEV)
    more = (torch.randn(8, H, generator=g) * 0.1).bfloat16()   # on the host: every append makes a device copy
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    one = (prompt.numel() + trail.numel() + more.numel()) * 2    # bytes one round hands the engine
    eng.session_begin(1, pad, _greedy(), max_trailing=64)
    codes = torch.zeros(1, 8, G, dtype=torch.int32, device=DEV)
    levels = []
    for _ in range(20):
        eng.admit([0], [0], [prompt], [trail])
        eng.append_trailing(0, more)
        eng.decode(4, codes)
        eng.release_slots([0])
        torch.cuda.synchronize()
        levels.append(torch.cuda.memory_allocated())
    eng.close()
    grown = max(levels) - levels[0]
    assert grown <= one, f"{grown} B kept over 20 admissions (one admission is {one} B)"


def test_scratch_growth_is_bounded():
    """Prefills with more prompt tokens, a larger trailing capacity and a larger batch each time: the engine frees the
    prefill scratch and the trailing buffer it outgrows, so it ends up holding the largest of each, not their sum."""
    cfg, Wb = _tiny()
    tc = cfg.talker
    eng = _engine(cfg, Wb, max_batch=32, max_ctx=1024)
    H = tc.hidden_size
    g = torch.Generator().manual_seed(1)
    prompts = (torch.randn(32, 1000, H, generator=g) * 0.5).bfloat16().to(DEV)
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    empty = torch.zeros(0, H, dtype=torch.bfloat16)
    sp = _greedy()

    def prefill(i):   # i = 1..8: a batch of 4i rows of 125i tokens, room for 512i trailing rows each
        B, n = 4 * i, 125 * i
        eng.prefill([prompts[b, :n] for b in range(B)], [empty] * B, pad, sp, trailing_capacity=512 * i)

    # the largest prefill (32 x 1000 tokens) and trailing buffer (4096 rows of the 32 slots): per token x, normed x,
    # qkv, attention output and MLP activation in bf16 plus sequence and position ids, for the 1.25x capacity the
    # engine reserves
    per_tok = 2 * (2 * H + (tc.num_heads + 2 * tc.num_kv_heads) * tc.head_dim + tc.num_heads * tc.head_dim
                   + tc.intermediate_size) + 8
    scratch = per_tok * (32000 + 32000 // 4)
    trailing = 32 * 4096 * H * 2
    slack = 32 * MiB   # up to 2 MiB of page rounding on each of the engine's scratch, trailing and program blocks
    assert scratch >= 4 * slack
    grown = _growth(prefill, list(range(1, 9)))
    eng.close()
    assert grown <= scratch + trailing + slack, \
        f"{grown / MiB:.0f} MiB kept after growing prefills (largest scratch {scratch / MiB:.0f} MiB, trailing {trailing / MiB:.0f} MiB)"


@pytest.mark.parametrize("case", ["missing", "half_norm", "qkv_rows"])
def test_tensor_errors_are_reported_at_finalize(monkeypatch, case):
    from qwen3_tts_b200.engine import AREngine
    cfg, Wb = _tiny()
    H, QKV = cfg.talker.hidden_size, (cfg.talker.num_heads + 2 * cfg.talker.num_kv_heads) * cfg.talker.head_dim
    put = AREngine._put

    def bad_put(self, name, x):
        if case == "missing" and name == "cp.norm":
            return
        if case == "half_norm" and name == "talker.layers.0.ln2":
            x = x.reshape(-1)[: H // 2]
        if case == "qkv_rows" and name == "talker.layers.0.qkv":
            x = x[:-16]
        put(self, name, x)

    load, loaded = AREngine._load, []

    def load_all(self, W):   # every tensor went in: what fails after this is q3_engine_finalize
        load(self, W)
        loaded.append(True)

    monkeypatch.setattr(AREngine, "_put", bad_put)
    monkeypatch.setattr(AREngine, "_load", load_all)
    with pytest.raises(RuntimeError) as err:
        _engine(cfg, Wb)
    msg = str(err.value)
    assert loaded, f"failed while loading, not at finalize: {msg}"
    assert "AR engine" in msg, msg
    if case == "missing":
        assert "cp.norm" in msg and "missing" in msg and str(cfg.cp.hidden_size) in msg, msg
    elif case == "half_norm":
        assert "talker.layers.0.ln2" in msg and str(H // 2) in msg and str(H) in msg, msg
    else:
        counts = str((QKV - 16) * H) in msg and str(QKV * H) in msg
        shapes = f"[{QKV - 16}][{H}]" in msg and f"[{QKV}][{H}]" in msg
        assert "talker.layers.0.qkv" in msg and (counts or shapes), msg


def test_failed_create_leaves_the_process_usable():
    """A max_ctx whose KV cache is tens of TB: cudaMalloc refuses it without reserving anything.  The constructor
    reports it, and neither torch's next kernel nor a fresh engine sees that error afterwards."""
    cfg, Wb = _tiny()
    embs, trail, pad = Hh.make_inputs(cfg, [6, 9], [2, 0], seed=7)
    before = _engine(cfg, Wb)
    want = before.generate(embs, trail, pad, _greedy())
    before.close()
    with pytest.raises(RuntimeError, match="cudaMalloc"):
        _engine(cfg, Wb, max_batch=32, max_ctx=1 << 30)
    x = torch.arange(1024, device=DEV, dtype=torch.float32)
    assert (x * 2).sum().item() == 1023 * 1024
    after = _engine(cfg, Wb)
    got = after.generate(embs, trail, pad, _greedy())
    after.close()
    assert all(torch.equal(a, b) for a, b in zip(got, want))
