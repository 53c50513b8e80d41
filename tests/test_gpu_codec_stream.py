"""Stateful streaming codec decoder (q3_codec_stream_*, SURVEY §8b / §8f-2) against the engine's own one-shot causal
forward and against the CPU oracle's streaming spec (oracle/codec.py::StreamingDecoder)."""
import dataclasses

import numpy as np
import pytest
import torch

from oracle import codec as OC
from tests.test_gpu_codec import _small_cfg, _pkg_cfg, _bf16_round, _snr_db

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("B,packets", [(1, [1, 1, 1, 1, 1, 1, 1, 1]), (2, [4, 4, 4, 4, 4]), (3, [3, 1, 5, 2, 8, 7, 4, 1, 6])])
def test_ragged_packets_equal_one_shot_forward_in_every_row(B, packets):
    """Packets of any sizes (window 6 < packet, window > packet, packet > every conv history) reproduce the one-shot
    forward of the same engine exactly, and the oracle's stateful spec within the codec tolerance."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    Wb, Wf = _bf16_round(OC.random_weights(cfg, seed=5))
    T = sum(packets)
    g = torch.Generator().manual_seed(6)
    codes = torch.randint(0, cfg.codebook_size, (B, cfg.num_quantizers, T), generator=g)
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=64)
    one = dec.forward(codes.to(DEV)).cpu()
    st = dec.open_stream(B, max_packet_frames=8)
    outs, s0 = [], 0
    for n in packets:
        outs.append(st.push(codes[:, :, s0:s0 + n].to(DEV)).cpu())
        s0 += n
    assert st.positions == [T] * B
    got = torch.cat(outs, -1)
    assert got.shape == one.shape == (B, 1, T * 1920)
    d = (got - one).abs().max().item()
    assert d == 0.0, f"stream differs from the one-shot forward by {d}"
    # the oracle's streaming decoder (fp32 on the same bf16-rounded weights), same ragged packets
    spec = OC.StreamingDecoder(Wf, cfg, batch=B)
    ref, s0 = [], 0
    for n in packets:
        ref.append(spec.push(codes[:, :, s0:s0 + n]))
        s0 += n
    ref = torch.cat(ref, -1)
    assert _snr_db(ref, got) > 25.0
    # a reset starts new utterances: the same codes give the same audio again
    st.reset()
    again = st.push(codes[:, :, :packets[0]].to(DEV)).cpu()
    assert torch.equal(again, outs[0])
    st.close()
    dec.close()


def test_full_config_stream_packets_of_4():
    """Default 195 M-parameter decoder, 4-frame packets (the report's 320 ms packet), 24 frames, B=2."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = OC.CodecCfg()
    Wb, Wf = _bf16_round(OC.random_weights(cfg, seed=1))
    B, T = 2, 24
    g = torch.Generator().manual_seed(2)
    codes = torch.randint(0, cfg.codebook_size, (B, cfg.num_quantizers, T), generator=g)
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=128)
    one = dec.forward(codes.to(DEV)).cpu()
    st = dec.open_stream(B, max_packet_frames=4)
    got = torch.cat([st.push(codes[:, :, s:s + 4].to(DEV)).cpu() for s in range(0, T, 4)], -1)
    assert (got - one).abs().max().item() == 0.0
    ref = OC.decoder_forward(Wf, cfg, codes)
    assert _snr_db(ref, got) > 22.0
    st.close()
    dec.close()


@pytest.mark.parametrize("layers,ok", [(27, True), (28, False)])
def test_open_bounds_history_buffers_by_the_roll_table(layers, ok):
    """One launch after every packet rolls all history buffers (pre, in, out, one K/V window per layer, one per
    upsampling stage, four per decoder block) from a table of 48 entries. Open accepts 3 + 27 + 2 + 16 = 48 buffers
    and refuses 49 with an error instead of overrunning the table. Open only: nothing is stepped."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = dataclasses.replace(_small_cfg(), num_layers=layers)
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=3))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=64)
    if ok:
        dec.open_stream(2, max_packet_frames=4).close()
    else:
        with pytest.raises(RuntimeError, match="49 history buffers"):
            dec.open_stream(2, max_packet_frames=4)
    dec.close()
