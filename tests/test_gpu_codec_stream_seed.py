"""Seeding rows of the streaming codec decoder with a reference prefix (CodecStream.seed, q3_codec_stream_copy_rows):
a seeded row continues exactly as the one-shot forward of cat(reference, continuation) does from the reference's end,
bit for bit, while the stream's other rows run on untouched."""
import ctypes as C
import re

import pytest
import torch

from oracle import codec as OC
from tests.test_gpu_codec import _small_cfg, _pkg_cfg, _bf16_round
from tests.test_gpu_codec_stream_rows import _garbage, _utt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UP = 1920


def _decoder(cfg, seed, max_frames):
    from qwen3_tts_b200.codec import CodecDecoder
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=seed))
    return CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=max_frames)


def _drive(st, n, todo, g):
    """Push ragged packets of n frames: todo[b] = codes (K, L) still to push for row b (None: idle).  Counts are drawn
    from {0 .. n}, with full packets mixed in.  Returns each row's audio."""
    B, K = st.B, st.dec.cfg.num_quantizers
    done, audio, step = [0] * B, [[] for _ in range(B)], 0
    while any(c is not None and done[b] < c.shape[1] for b, c in enumerate(todo)):
        counts, pkt = [0] * B, _garbage((B, K, n), g)
        for b, c in enumerate(todo):
            if c is None:
                continue
            k = min(int(torch.randint(0, n + 1, (1,), generator=g)), c.shape[1] - done[b])
            if step % 2 == b % 2:
                k = min(n, c.shape[1] - done[b])
            counts[b] = k
            pkt[b, :, :k] = c[:, done[b]:done[b] + k]
        wav = st.push(pkt.to(DEV), counts)[:, 0].cpu()
        for b in range(B):
            audio[b].append(wav[b, :counts[b] * UP])
            done[b] += counts[b]
        step += 1
    return [torch.cat(a) if a else torch.zeros(0) for a in audio]


def _one_shot(dec, codes):
    return dec.forward(codes[None].to(DEV))[0, 0].cpu()


def _seed_next_to_running_rows(cfg, dec, ref_lens, cont, g):
    """B = 4, 4-frame packets.  Rows 0 and 2 start plain utterances and run a few packets; then rows 1 and 3 are
    seeded with references (one call), later row 2 (running) is seeded in a second call, and everything is pushed out."""
    st = dec.open_stream(4, max_packet_frames=4)
    plain = {0: _utt(cfg, 30, g), 2: _utt(cfg, 9, g)}
    refs = [_utt(cfg, L, g).T for L in ref_lens]            # (L, K), the layout of ref_code
    conts = [_utt(cfg, cont, g) for _ in ref_lens]
    st.reset()
    head = _drive(st, 4, [plain[0][:, :10], None, plain[2], None], g)
    st.seed([1, 3], [refs[0], refs[1]])
    assert st.positions == [10, ref_lens[0], 9, ref_lens[1]]
    st.seed([2], [refs[2]])                                 # row 2 was running: the seed replaces it whole
    assert st.positions == [10, ref_lens[0], ref_lens[2], ref_lens[1]]
    tail = _drive(st, 4, [plain[0][:, 10:], conts[0], conts[2], conts[1]], g)
    assert torch.equal(torch.cat([head[0], tail[0]]), _one_shot(dec, plain[0]))
    assert torch.equal(head[2], _one_shot(dec, plain[2]))
    for row, i in ((1, 0), (3, 1), (2, 2)):
        L = ref_lens[i]
        want = _one_shot(dec, torch.cat([refs[i].T, conts[i]], 1))[L * UP:]
        assert tail[row].shape == want.shape
        d = (tail[row] - want).abs().max().item()
        assert d == 0.0, f"row {row} (reference of {L} frames) differs from forward(cat(ref, cont)) by {d}"
    st.close()


def test_seed_small_config():
    cfg = _small_cfg()
    dec = _decoder(cfg, 11, 128)
    g = torch.Generator().manual_seed(12)
    _seed_next_to_running_rows(cfg, dec, (5, 40, 80), 13, g)
    _seed_next_to_running_rows(cfg, dec, (1, 33, 7), 6, g)
    dec.close()


def test_seed_full_config_past_the_window_and_the_seed_packet():
    """Default decoder: references of 1, 5, 40 and 80 frames, so the K/V window (71 rows) and the 32-frame packet of
    the private seed stream are both exceeded."""
    cfg = OC.CodecCfg()
    dec = _decoder(cfg, 1, 128)
    g = torch.Generator().manual_seed(2)
    _seed_next_to_running_rows(cfg, dec, (40, 80, 5), 14, g)
    st = dec.open_stream(2, max_packet_frames=4)
    ref, cont = _utt(cfg, 1, g).T, _utt(cfg, 9, g)
    st.seed([0], [ref])
    got = _drive(st, 4, [cont, None], g)[0]
    assert torch.equal(got, _one_shot(dec, torch.cat([ref.T, cont], 1))[UP:])
    st.close()
    dec.close()


def test_seed_running_row_equals_reset_then_seed_and_one_call_equals_two():
    cfg = _small_cfg()
    dec = _decoder(cfg, 3, 96)
    g = torch.Generator().manual_seed(4)
    refs = [_utt(cfg, L, g).T for L in (12, 37)]
    conts = [_utt(cfg, 10, g) for _ in refs]
    warm = _utt(cfg, 8, g)
    a, b = dec.open_stream(3, max_packet_frames=4), dec.open_stream(3, max_packet_frames=4)
    for st in (a, b):
        st.push(torch.stack([warm] * 3).to(DEV))            # every row mid-utterance at position 8
    a.seed([0, 2], refs)                                    # one call over running rows
    b.reset([0, 2])
    b.seed([2], refs[1:])                                   # reset, then two calls in the other order
    b.seed([0], refs[:1])
    assert a.positions == b.positions == [12, 8, 37]
    wa = _drive(a, 4, [conts[0], None, conts[1]], torch.Generator().manual_seed(5))
    wb = _drive(b, 4, [conts[0], None, conts[1]], torch.Generator().manual_seed(5))
    assert all(torch.equal(x, y) for x, y in zip(wa, wb))
    a.close(), b.close()
    dec.close()


def test_copy_rows_forks_and_bridges_streams_of_different_shapes():
    """Through the C ABI: a source row listed twice gives two identical destination rows, and a 2-row stream with
    8-frame packets feeds a 3-row stream with 4-frame packets."""
    cfg = _small_cfg()
    dec = _decoder(cfg, 5, 64)
    lib = dec.lib
    g = torch.Generator().manual_seed(6)
    src, dst = dec.open_stream(2, max_packet_frames=8), dec.open_stream(3, max_packet_frames=4)
    pre = [_utt(cfg, 19, g), _utt(cfg, 11, g)]
    pkt = torch.zeros(2, cfg.num_quantizers, 19, dtype=torch.int32)
    pkt[0], pkt[1, :, :11] = pre[0], pre[1]
    src.push(pkt.to(DEV), [19, 11])
    dst.push(_utt(cfg, 4, g)[None].expand(3, -1, -1).contiguous().to(DEV))
    strm = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.q3_codec_stream_copy_rows(dst.h, src.h, 3, (C.c_int32 * 3)(0, 0, 1), (C.c_int32 * 3)(2, 0, 1), strm)
    assert rc == 0, lib.q3_last_error()
    assert dst.positions == [19, 11, 19] and src.positions == [19, 11]
    cont = _utt(cfg, 9, g)
    out = _drive(dst, 4, [cont, cont, cont], g)
    assert torch.equal(out[0], out[2])
    assert torch.equal(out[0], _one_shot(dec, torch.cat([pre[0], cont], 1))[19 * UP:])
    assert torch.equal(out[1], _one_shot(dec, torch.cat([pre[1], cont], 1))[11 * UP:])
    src.close(), dst.close()
    dec.close()


def test_invalid_arguments_change_nothing():
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    dec = _decoder(cfg, 7, 32)
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=7))
    other = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=32)
    lib = dec.lib
    g = torch.Generator().manual_seed(8)
    a, b = dec.open_stream(3, max_packet_frames=4), dec.open_stream(2, max_packet_frames=4)
    foreign = other.open_stream(3, max_packet_frames=4)
    utts = [_utt(cfg, 15, g) for _ in range(3)]
    head = _drive(a, 4, [u[:, :6] for u in utts], g)
    b.push(_utt(cfg, 5, g)[None].expand(2, -1, -1).contiguous().to(DEV))
    strm = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    i3 = lambda *v: (C.c_int32 * len(v))(*v)  # noqa: E731

    def copy(dst, src, n, s, d):
        return lib.q3_codec_stream_copy_rows(dst, src, n, s, d, strm)

    cases = [
        (lambda: copy(None, b.h, 1, i3(0), i3(0)), "null stream"),
        (lambda: copy(a.h, None, 1, i3(0), i3(0)), "null stream"),
        (lambda: copy(a.h, a.h, 1, i3(0), i3(1)), "same stream"),
        (lambda: copy(a.h, foreign.h, 1, i3(0), i3(1)), "different codecs"),
        (lambda: copy(a.h, b.h, -1, i3(0), i3(0)), "-1 rows to copy"),
        (lambda: copy(a.h, b.h, 4, i3(0, 0, 0, 0), i3(0, 1, 2, 0)), "4 rows to copy, the destination stream has 3"),
        (lambda: copy(a.h, b.h, 1, None, i3(0)), "null argument"),
        (lambda: copy(a.h, b.h, 2, i3(0, 2), i3(0, 1)), "source row 2 out of range \\[0, 2\\)"),
        (lambda: copy(a.h, b.h, 2, i3(0, -1), i3(0, 1)), "source row -1 out of range"),
        (lambda: copy(a.h, b.h, 2, i3(0, 1), i3(0, 3)), "destination row 3 out of range \\[0, 3\\)"),
        (lambda: copy(a.h, b.h, 2, i3(0, 1), i3(1, 1)), "destination row 1 listed twice"),
    ]
    for call, msg in cases:
        assert call() != 0, msg
        assert re.search(msg, lib.q3_last_error().decode()), (msg, lib.q3_last_error())
        assert a.positions == [6, 6, 6] and b.positions == [5, 5]
    assert copy(a.h, b.h, 0, None, None) == 0
    ok = _utt(cfg, 3, g).T
    bad = [
        (lambda: a.seed([0], [ok[:, :-1]]), "expected an \\(L, 16\\) tensor"),
        (lambda: a.seed([0], [ok.float()]), "integer codes"),
        (lambda: a.seed([0], [ok[:0]]), "0 frames outside \\[1, 32\\]"),
        (lambda: a.seed([0], [_utt(cfg, 33, g).T]), "33 frames outside \\[1, 32\\]"),
        (lambda: a.seed([0], [ok - 1 - ok.max()]), "codes must lie in \\[0, 64\\)"),
        (lambda: a.seed([0], [ok + cfg.codebook_size]), "codes must lie in \\[0, 64\\)"),
        (lambda: a.seed([3], [ok]), "seed row 3 out of range"),
        (lambda: a.seed([1, 1], [ok, ok]), "not distinct"),
        (lambda: a.seed([0, 1], [ok]), "2 rows for 1"),
    ]
    for call, msg in bad:
        with pytest.raises(ValueError, match=msg):
            call()
        assert a.positions == [6, 6, 6]
    assert a._seeder is None                              # nothing was opened, let alone launched
    tail = _drive(a, 4, [u[:, 6:] for u in utts], g)
    for u, h, t in zip(utts, head, tail):
        assert torch.equal(torch.cat([h, t]), _one_shot(dec, u))
    for s in (a, b, foreign):
        s.close()
    other.close()
    dec.close()
