"""Streaming codec encoder (q3_codec_enc_stream_*, EncoderStream): the codes of a clip pushed in chunks of any sizes and
ended with end() equal, bit for bit, the GPU one-shot encode of that clip alone (B = 1), which test_gpu_codec_encoder.py
pins to the oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mimi_encoder as M

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HOP = 1920
CHUNKS = [1, 37, 959, 1919, 1920, 1921, 3 * 1920, 9 * 1920]


def _tiny(max_frames=512, seed=3):
    from qwen3_tts_b200.codec_encoder import CodecEncoder
    from tests.test_gpu_codec_encoder import _pkg_cfg
    cfg = M.cfg_tiny_encoder()
    return CodecEncoder(_pkg_cfg(cfg), M.random_weights(cfg, seed=seed), device=DEV, max_frames=max_frames)


_TOK = []


def _tokenizer():
    """Default encoder config with seeded random weights, behind the product wrapper (built once per module)."""
    if not _TOK:
        import qwen3_tts_b200 as q
        from qwen3_tts_b200 import synthetic
        from qwen3_tts_b200.config import EncoderConfig
        from qwen3_tts_b200.model import Qwen3TTSTokenizer
        ecfg, ccfg = EncoderConfig(), q.CodecConfig()
        _TOK.append(Qwen3TTSTokenizer(ccfg, synthetic.random_codec_weights(ccfg, device=DEV, seed=1), device=DEV, max_frames=64,
                                      encoder_cfg=ecfg, encoder_weights=synthetic.random_encoder_weights(ecfg, seed=2)))
    return _TOK[0]


def _clip(n, seed):
    g = np.random.default_rng(seed)
    return np.clip(g.standard_normal(n).astype(np.float32) * 0.1, -1, 1)


def _solo(enc, clip):
    return enc.encode([torch.from_numpy(clip)])[0].cpu()


def _stream_clip(st, row, clip, sizes):
    got, i, k = [], 0, 0
    while i < len(clip):
        n = sizes[k % len(sizes)]
        got.append(st.push({row: clip[i: i + n]})[row].cpu())
        i, k = i + n, k + 1
    got.append(st.end([row])[row].cpu())
    return torch.cat(got)


@pytest.mark.parametrize("length", [1, 1919, 1920, 1921, 10 * HOP, 10 * HOP + 7])
def test_lengths_and_chunkings_equal_one_shot(length):
    tok = _tokenizer()
    clip = _clip(length, length)
    want = tok.encode(clip, sr=24000).audio_codes[0].cpu()
    st = tok.open_encode_stream(batch=1, max_packet_frames=8)
    rng = np.random.default_rng(length)
    plans = [[c] for c in CHUNKS if length // c <= 200] + [list(rng.choice(CHUNKS[1:], size=16))]
    for sizes in plans:
        got = _stream_clip(st, 0, clip, sizes)
        assert got.shape == want.shape and torch.equal(got, want), f"chunks {sizes}"
        assert st.positions == [0]
    st.close()


def test_one_shot_rows_of_a_batch_equal_their_solo_encodes():
    """The one-shot runs through the same walker as the stream: at the default shapes (MLP hidden wider than qkv) every
    row of a batch equals its solo encode (whole-frame clips: right padding changes the last frame of any other)."""
    tok = _tokenizer()
    clips = [_clip(n, n) for n in (3 * HOP, 5 * HOP + 11, 2 * HOP)]
    rows = tok.encode(clips, sr=24000).audio_codes
    for clip, got in zip(clips, rows):
        assert torch.equal(got.cpu(), tok.encode(clip, sr=24000).audio_codes[0].cpu())


def test_staggered_rows_equal_their_solo_clips():
    enc = _tiny()
    st = enc.open_stream(5, max_packet_frames=4)
    rng = np.random.default_rng(11)
    # per row: list of (start step, clip length); rows idle between and before clips
    plan = {0: [(0, 7 * HOP + 100), (9, 3 * HOP)], 1: [(2, 5 * HOP + 1919)], 2: [(1, 1500), (4, 9 * HOP + 3)],
            3: [(5, 4 * HOP)], 4: [(0, 11 * HOP + 960)]}
    queue = {b: [(s, _clip(n, 100 * b + s)) for s, n in v] for b, v in plan.items()}
    cur = {b: None for b in plan}   # [clip, offset, codes so far]
    done = {b: [] for b in plan}
    for step in range(80):
        if step == 6:   # a reset between pushes: row 3's clip is dropped and restarted, its neighbours carry on
            st.reset([3])
            if cur[3] is not None:
                cur[3] = [cur[3][0], 0, []]
        push, ending = {}, []
        for b in plan:
            if cur[b] is None and queue[b] and queue[b][0][0] <= step:
                cur[b] = [queue[b].pop(0)[1], 0, []]
            if cur[b] is None:
                continue
            clip, off, _ = cur[b]
            if off >= len(clip):
                ending.append(b)
            elif rng.random() < 0.7:   # otherwise the row idles this step
                n = int(rng.choice(CHUNKS[1:7]))
                push[b] = clip[off: off + n]
                cur[b][1] = off + n
        out = st.push(push) if push else {}
        for b, c in out.items():
            cur[b][2].append(c.cpu())
        if ending:
            for b, c in st.end(ending).items():
                cur[b][2].append(c.cpu())
                done[b].append((cur[b][0], torch.cat(cur[b][2])))
                cur[b] = None
    for b in plan:
        assert len(done[b]) == len(plan[b]), f"row {b} finished {len(done[b])} clips"
        for clip, got in done[b]:
            assert torch.equal(got, _solo(enc, clip)), f"row {b}, clip of {len(clip)} samples"
    st.close()


def test_tiny_window_many_frames_and_packet_sizes():
    enc = _tiny()
    clip = _clip(40 * HOP + 333, 5)   # 81 transformer frames, window 6
    want = _solo(enc, clip)
    for mpf, sizes in ((1, [HOP]), (3, [5 * HOP + 17]), (8, [9 * HOP, 37])):
        st = enc.open_stream(2, max_packet_frames=mpf)
        assert torch.equal(_stream_clip(st, 1, clip, sizes), want), (mpf, sizes)
        st.close()


def test_default_config_12s_past_the_window():
    tok = _tokenizer()
    clip = _clip(12 * 24000, 12)   # 300 transformer frames > window 250
    want = tok.encode(clip, sr=24000).audio_codes[0].cpu()
    st = tok.open_encode_stream(batch=2, max_packet_frames=4)
    got = _stream_clip(st, 1, clip, [4 * HOP])
    assert torch.equal(got, want)
    st.close()


def test_replicate_edge_first_packet_single_frame_and_sub_frame_clip():
    enc = _tiny()
    st = enc.open_stream(3, max_packet_frames=4)
    clip = _clip(6 * HOP + 50, 21)
    got = [st.push({0: clip[:HOP]})[0].cpu()]          # the row's first packet is one frame
    assert got[0].shape[0] == 1
    got.append(st.push({0: clip[HOP:]})[0].cpu())
    got.append(st.end([0])[0].cpu())
    assert torch.equal(torch.cat(got), _solo(enc, clip))
    for n in (1, 700, HOP - 1):                         # shorter than one frame: only end() encodes
        short = _clip(n, n)
        assert st.push({2: short})[2].shape == (0, 16)
        last = st.end([2])[2].cpu()
        assert last.shape == (1, 16) and torch.equal(last, _solo(enc, short))
    st.close()


def test_position_limit_rejects_without_moving_positions():
    enc = _tiny(max_frames=10)   # 10 transformer frames = 5 codec frames per clip
    st = enc.open_stream(2, max_packet_frames=4)
    st.push({0: _clip(4 * HOP, 1), 1: _clip(2 * HOP, 2)})
    assert st.positions == [4, 2]
    with pytest.raises(ValueError, match="row 0"):
        st.push({0: _clip(2 * HOP, 3), 1: _clip(HOP, 4)})
    assert st.positions == [4, 2]
    st.push({0: _clip(HOP, 5)})
    assert st.positions == [5, 2]
    # the clip is full: a non-empty tail would pass the RoPE table too
    st.push({0: _clip(10, 6)})
    with pytest.raises(RuntimeError, match="row 0"):
        st.end([0])
    assert st.positions == [5, 2]
    # the native check on its own (the Python one bypassed)
    counts = (C.c_int32 * 2)(1, 0)
    wav = torch.zeros(2, HOP, device=DEV)
    codes = torch.empty(2, 16, 1, dtype=torch.int32, device=DEV)
    rc = st.lib.q3_codec_enc_stream_step_rows(st.h, wav.data_ptr(), 1, counts, codes.data_ptr(), None)
    assert rc != 0 and "row 0" in st.lib.q3_last_error().decode()
    assert st.positions == [5, 2]
    st.close()


def test_argument_checks_change_no_position():
    enc = _tiny()
    st = enc.open_stream(3, max_packet_frames=2)
    st.push({0: _clip(HOP, 1), 1: _clip(2 * HOP, 2)})
    before = st.positions
    lib, h = st.lib, st.h
    wav = torch.zeros(3, 3 * HOP, device=DEV)
    codes = torch.empty(3, 16, 3, dtype=torch.int32, device=DEV)
    i32 = C.c_int32

    def err():
        return lib.q3_last_error().decode()

    assert lib.q3_codec_enc_stream_step_rows(h, wav.data_ptr(), 2, (i32 * 3)(1, 3, 0), codes.data_ptr(), None) != 0
    assert "row 1" in err()
    assert lib.q3_codec_enc_stream_step_rows(h, wav.data_ptr(), 2, (i32 * 3)(0, 0, -1), codes.data_ptr(), None) != 0
    assert "row 2" in err()
    assert lib.q3_codec_enc_stream_step_rows(h, wav.data_ptr(), 3, (i32 * 3)(1, 1, 1), codes.data_ptr(), None) != 0
    assert lib.q3_codec_enc_stream_step_rows(h, None, 1, (i32 * 3)(1, 1, 1), codes.data_ptr(), None) != 0
    assert lib.q3_codec_enc_stream_step_rows(h, wav.data_ptr(), 1, (i32 * 3)(1, 1, 1), None, None) != 0
    fin = lambda n, rows, tails: lib.q3_codec_enc_stream_finish_rows(  # noqa: E731
        h, n, (i32 * len(rows))(*rows), (i32 * len(tails))(*tails), wav.data_ptr(), codes.data_ptr(), None)
    assert fin(1, [0], [HOP]) != 0 and "row 0" in err()
    assert fin(1, [1], [-1]) != 0 and "row 1" in err()
    assert fin(1, [3], [5]) != 0 and "row 3" in err()
    assert fin(2, [1, 1], [5, 5]) != 0 and "row 1" in err()
    assert lib.q3_codec_enc_stream_reset_rows(h, 2, (i32 * 2)(2, 2), None) != 0 and "row 2" in err()
    assert lib.q3_codec_enc_stream_reset_rows(h, 1, (i32 * 1)(-1), None) != 0 and "row -1" in err()
    assert lib.q3_codec_enc_stream_row_position(h, 3) == -1
    assert st.positions == before
    # Python level
    for bad in ({5: _clip(10, 1)}, {0: np.zeros((2, 10), np.float32)}, {1: np.array([0.0, np.nan], np.float32)},
                {0: torch.tensor([np.inf])}, [np.zeros(10, np.float32)]):
        with pytest.raises(ValueError):
            st.push(bad)
    for bad in ([3], [0, 0], [-1]):
        with pytest.raises(ValueError):
            st.end(bad)
        with pytest.raises(ValueError):
            st.reset(bad)
    assert st.positions == before
    st.close()


def test_decode_only_tokenizer_refuses_a_stream():
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.model import Qwen3TTSTokenizer
    ccfg = q.CodecConfig()
    tok = Qwen3TTSTokenizer(ccfg, synthetic.random_codec_weights(ccfg, device=DEV, seed=1), device=DEV, max_frames=16)
    with pytest.raises(RuntimeError, match="decode-only"):
        tok.open_encode_stream()


def test_stream_memory_matches_state_table_and_does_not_accumulate():
    from tests.test_gpu_scratch_growth import MiB, SLACK, _process_bytes
    from qwen3_tts_b200.config import EncoderConfig
    tok = _tokenizer()
    enc = tok.encoder
    cfg = EncoderConfig()
    # history per row (fp32), from the state table: waveform, per ratio x and z (max(k3 - 1, ratio) columns each at the
    # block's rate), conv_last's input, the residual stream for the downsample, and each layer's K/V window; plus the
    # history-prefixed buffers' packet capacity
    n = 4
    cap, c = n * HOP, cfg.num_filters
    per_row = (cfg.kernel_size - 1 + cap) * 1
    for r in cfg.ratios:
        per_row += 2 * c * (max(cfg.residual_kernel_size - 1, r) + cap)
        cap //= r
        c *= 2
    per_row += c * (cfg.last_kernel_size - 1 + cap) + cfg.hidden_size * (cfg.downsample_stride + cap)
    per_row += cfg.num_layers * 2 * cfg.hidden_size * (cfg.sliding_window - 1 + cap)
    per_row *= 4
    kv_state = cfg.num_layers * 2 * cfg.hidden_size * (cfg.sliding_window - 1) * 4
    assert 7 * MiB < kv_state < 8 * MiB   # the K/V windows dominate: ~7.8 MiB per row
    st = enc.open_stream(1, max_packet_frames=n)   # the packet scratch (the encoder's, shared) reaches its B = 32 size below
    st.close()
    big = enc.open_stream(32, max_packet_frames=n)
    big.close()
    torch.cuda.synchronize()
    m0, r0 = _process_bytes(), torch.cuda.memory_reserved()
    for _ in range(3):
        s = enc.open_stream(32, max_packet_frames=n)
        s.push({b: _clip(HOP, b) for b in range(32)})
        torch.cuda.synchronize()
        held = (_process_bytes() - m0) - (torch.cuda.memory_reserved() - r0)
        pages = (2 * len(cfg.ratios) + 5 + cfg.num_layers) * 2 * MiB   # each history buffer rounds up to 2 MiB pages
        assert 32 * per_row - SLACK <= held <= 32 * per_row + pages + SLACK, \
            f"stream holds {held / MiB:.0f} MiB, state table says {32 * per_row / MiB:.0f} MiB"
        s.close()
    torch.cuda.synchronize()
    grown = (_process_bytes() - m0) - (torch.cuda.memory_reserved() - r0)
    assert grown <= SLACK, f"{grown / MiB:.0f} MiB kept after closing streams"
