"""Per-row state of the streaming codec decoder (q3_codec_stream_step_rows / reset_rows / row_position): rows that
start, stop and restart at different frames share one stream, and every utterance's audio equals the one-shot forward
of its codes alone (B = 1) bit for bit."""
import ctypes as C
import re

import pytest
import torch

from oracle import codec as OC
from tests.test_gpu_codec import _small_cfg, _pkg_cfg, _bf16_round

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UP = 1920


def _garbage(shape, g):
    """codes that must never be read: -1 and values far outside the codebook"""
    return torch.where(torch.rand(shape, generator=g) < 0.5, torch.full(shape, -1), torch.full(shape, 1 << 20)).to(torch.int32)


def _session(dec, st, n, plan, g):
    """Drive `st` (B rows, packets of n frames) through `plan`: plan[b] is a list of (start_step, codes (K, L), keep)
    per row; at start_step the row is reset and its utterance starts; `keep` frames of it are pushed (keep < L
    abandons it, as a request released mid-utterance).  Counts are drawn from {0, 1 .. n} per step.  Checks the zero
    tails and the positions after every step; returns {(b, i): (codes pushed, audio)} and the positions of all rows
    before every reset."""
    B, K = st.B, dec.cfg.num_quantizers
    queue = [list(p) for p in plan]
    cur = [None] * B                      # (utterance key, codes, keep, frames pushed)
    audio, pos, step, at_resets = {}, [0] * B, 0, []
    while any(queue) or any(c is not None for c in cur):
        resets = []
        for b in range(B):
            if queue[b] and queue[b][0][0] <= step and cur[b] is None:
                _, codes, keep = queue[b].pop(0)
                cur[b] = [(b, len(plan[b]) - len(queue[b]) - 1), codes, keep, 0]
                resets.append(b)
                pos[b] = 0
        if resets:
            at_resets.append(st.positions)
            st.reset(resets)
        counts = [0] * B
        pkt = _garbage((B, K, n), g)
        for b in range(B):
            if cur[b] is None:
                continue
            key, codes, keep, done = cur[b]
            k = min(int(torch.randint(0, n + 1, (1,), generator=g)), keep - done)
            if step % 3 == b % 3:
                k = min(n, keep - done)   # every row also takes full packets
            counts[b] = k
            pkt[b, :, :k] = codes[:, done:done + k]
        wav = st.push(pkt.to(DEV), counts)[:, 0].cpu()
        for b in range(B):
            k = counts[b]
            assert (wav[b, k * UP:] == 0).all(), f"row {b}: audio past its count {k} at step {step}"
            pos[b] += k
            if cur[b] is None:
                continue
            key = cur[b][0]
            audio.setdefault(key, [cur[b][1], []])[1].append(wav[b, :k * UP])
            cur[b][3] += k
            if cur[b][3] == cur[b][2]:
                cur[b] = None
        assert st.positions == pos, (step, st.positions, pos)
        step += 1
    return {k: (c[:, :sum(a.shape[0] for a in w) // UP], torch.cat(w)) for k, (c, w) in audio.items()}, at_resets


def _check_solo(dec, got):
    for key, (codes, wav) in got.items():
        ref = dec.forward(codes[None].to(DEV))[0, 0].cpu()
        assert wav.shape == ref.shape, (key, wav.shape, ref.shape)
        d = (wav - ref).abs().max().item() if wav.numel() else 0.0
        assert d == 0.0, f"utterance {key} differs from its solo one-shot forward by {d}"


def _utt(cfg, L, g):
    return torch.randint(0, cfg.codebook_size, (cfg.num_quantizers, L), generator=g)


def test_rows_start_stop_and_reset_independently():
    """B = 3, 4-frame packets: rows start at different packets, row 2 is reset twice mid-session (one utterance is
    abandoned part-way), counts mix 0, < n and n; rows 0 and 1 run across row 2's resets untouched."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=7))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=64)
    g = torch.Generator().manual_seed(8)
    plan = [[(0, _utt(cfg, 30, g), 30)],
            [(2, _utt(cfg, 17, g), 17), (9, _utt(cfg, 9, g), 9)],
            [(1, _utt(cfg, 5, g), 5), (3, _utt(cfg, 20, g), 11), (6, _utt(cfg, 8, g), 8)]]
    st = dec.open_stream(3, max_packet_frames=4)
    got, _ = _session(dec, st, 4, plan, g)
    assert len(got) == 6 and got[(2, 1)][0].shape[1] == 11
    _check_solo(dec, got)
    st.close()
    dec.close()


def test_full_config_rows_staggered_past_the_window():
    """Default 195 M-parameter decoder, B = 4, 4-frame packets, max_frames = 128: row starts spread over more than the
    72-frame attention window and >= 90 frames per row, so rows attend at positions on both sides of the window while
    their neighbours start fresh."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = OC.CodecCfg()
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=1))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=128)
    g = torch.Generator().manual_seed(4)
    plan = [[(s, _utt(cfg, L, g), L)] for s, L in ((0, 96), (9, 92), (18, 100), (30, 90))]
    st = dec.open_stream(4, max_packet_frames=4)
    got, at_resets = _session(dec, st, 4, plan, g)
    assert sorted(got) == [(b, 0) for b in range(4)]
    assert max(at_resets[-1]) > cfg.sliding_window, at_resets  # the last row starts after row 0 has left its window
    _check_solo(dec, got)
    st.close()
    dec.close()


def test_push_without_counts_equals_every_count_n():
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=2))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=64)
    g = torch.Generator().manual_seed(3)
    codes = torch.randint(0, cfg.codebook_size, (2, cfg.num_quantizers, 19), generator=g).to(DEV)
    a, b = dec.open_stream(2, max_packet_frames=4), dec.open_stream(2, max_packet_frames=4)
    for s0, n in ((0, 3), (3, 4), (7, 12)):   # the last push is cut into packets of 4, 4, 4
        wa = a.push(codes[:, :, s0:s0 + n]).cpu()
        wb = b.push(codes[:, :, s0:s0 + n], counts=[n, n]).cpu()
        assert torch.equal(wa, wb)
    assert a.positions == b.positions == [19, 19]
    a.close(), b.close()
    dec.close()


def test_row_parked_at_the_table_end_takes_count_zero():
    """A row at position max_frames takes count 0 while the other rows step: accepted, and the others stay exact."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=9))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=16)
    g = torch.Generator().manual_seed(10)
    u0, u1 = _utt(cfg, 16, g), _utt(cfg, 14, g)
    st = dec.open_stream(2, max_packet_frames=4)
    w1 = []
    for s0 in range(0, 16, 4):
        pkt = _garbage((2, cfg.num_quantizers, 4), g)
        pkt[0], k1 = u0[:, s0:s0 + 4], min(4, max(0, 6 - s0))
        pkt[1, :, :k1] = u1[:, s0:s0 + k1]
        w1.append(st.push(pkt.to(DEV), [4, k1])[1, 0, :k1 * UP].cpu())
    assert st.positions == [16, 6]
    for s0 in range(6, 14, 4):                       # row 0 is parked at max_frames = 16
        pkt = _garbage((2, cfg.num_quantizers, 4), g)
        pkt[1] = u1[:, s0:s0 + 4]
        wav = st.push(pkt.to(DEV), [0, 4])[:, 0].cpu()
        assert (wav[0] == 0).all()
        w1.append(wav[1])
    assert st.positions == [16, 14]
    ref = dec.forward(u1[None].to(DEV))[0, 0].cpu()
    assert torch.equal(torch.cat(w1), ref)
    st.close()
    dec.close()


def test_argument_checks_name_the_row_and_change_no_position():
    """Every check fires before any device work.  Each bad case is paired with n = 0 (step) or more rows than the
    stream has (reset), so that a later check would refuse the call anyway and nothing is launched without it."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=5))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=8)
    lib = dec.lib
    st = dec.open_stream(3, max_packet_frames=4)
    g = torch.Generator().manual_seed(6)
    st.push(torch.randint(0, cfg.codebook_size, (3, cfg.num_quantizers, 4), generator=g).to(DEV), [4, 2, 0])
    st.push(torch.randint(0, cfg.codebook_size, (3, cfg.num_quantizers, 4), generator=g).to(DEV), [4, 0, 1])
    assert st.positions == [8, 2, 1]
    codes = torch.zeros(3, cfg.num_quantizers, 4, dtype=torch.int32, device=DEV)
    wav = torch.zeros(3, 4 * UP, device=DEV)
    strm = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def step(counts, n=0, c=codes.data_ptr(), w=wav.data_ptr()):
        return lib.q3_codec_stream_step_rows(st.h, c, n, (C.c_int32 * 3)(*counts), w, strm)

    def reset(rows, n=None):
        return lib.q3_codec_stream_reset_rows(st.h, len(rows) if n is None else n, (C.c_int32 * len(rows))(*rows), strm)

    cases = [
        (lambda: step([0, 0, 0], c=None), "null argument"),
        (lambda: step([0, 0, 0], w=None), "null argument"),
        (lambda: step([0, -1, 0]), "row 1: count -1 outside \\[0, 0\\]"),
        (lambda: step([0, 0, 1]), "row 2: count 1 outside \\[0, 0\\]"),
        (lambda: step([1, 0, 0]), "row 0: position 8 \\+ 1 frames exceeds the RoPE table \\(max_frames 8\\)"),
        (lambda: step([0, 0, 0]), "packet of 0 frames"),
        (lambda: reset([0, 1, 2, 3]), "reset row 3 out of range \\[0, 3\\)"),
        (lambda: reset([0, 1, 1, 2]), "reset row 1 listed twice"),
        (lambda: reset([-1, 0, 1, 2]), "reset row -1 out of range"),
        (lambda: lib.q3_codec_stream_reset_rows(st.h, 0, None, strm), "null argument"),
    ]
    for call, msg in cases:
        assert call() != 0, msg
        assert re.search(msg, lib.q3_last_error().decode()), (msg, lib.q3_last_error())
        assert st.positions == [8, 2, 1]
    assert lib.q3_codec_stream_row_position(st.h, 3) == -1 and "row 3 out of range" in lib.q3_last_error().decode()
    with pytest.raises(ValueError, match="row 1: count 5 outside"):
        st.push(codes, [0, 5, 0])
    # the stream still works: reset one row, the others keep their positions
    st.reset([0])
    assert st.positions == [0, 2, 1]
    st.close()
    dec.close()
