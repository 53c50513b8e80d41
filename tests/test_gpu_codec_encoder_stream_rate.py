"""The streaming encoder at another input rate (open_encode_stream(sample_rate=)): ragged pushes plus end equal
CodecEncoder.forward of Resampler.oneshot of the clip, bit for bit, for several rows with different clip lengths."""
import numpy as np
import pytest
import torch

from tests.test_gpu_codec_encoder_stream import _clip, _tokenizer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [1, 0, 333, 1279, 5000, 17, 640, 2560]


@pytest.mark.parametrize("rate", [16000, 48000])
def test_resampled_stream_equals_forward_of_oneshot(rate):
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.audio import Resampler
    tok = _tokenizer()
    lengths = [rate // 10 + 1, 3 * 1920 * rate // 24000 + 5, 7 * rate // 12 + 3]
    clips = [_clip(n, 17 * i + rate) for i, n in enumerate(lengths)]
    st = tok.open_encode_stream(batch=len(clips), max_packet_frames=4, sample_rate=rate)
    got = {r: [] for r in range(len(clips))}
    off = [0] * len(clips)
    for k in range(200):
        push = {}
        for r, c in enumerate(clips):
            if off[r] < len(c):
                n = SIZES[(k + 2 * r) % len(SIZES)]
                push[r] = c[off[r]: off[r] + n]
                off[r] += len(push[r])
        if not push:
            break
        for r, codes in st.push(push).items():
            got[r].append(codes.cpu())
    for r, codes in st.end(list(range(len(clips)))).items():
        got[r].append(codes.cpu())
    res = Resampler(DEV, 1, 64)
    for r, c in enumerate(clips):
        wav = torch.from_numpy(res.oneshot(c, rate, AudioFormat(24000)))
        want = tok.encoder.forward(wav[None].to(DEV))[0].T.cpu()
        have = torch.cat(got[r])
        assert have.shape == want.shape and torch.equal(have, want), (rate, r, have.shape, want.shape)
    # a reset row starts a new clip at position 0 of both the resampler and the encoder
    st.push({0: clips[0][:999]})
    st.reset([0])
    codes = [st.push({0: clips[1]})[0].cpu(), st.end([0])[0].cpu()]
    wav = torch.from_numpy(res.oneshot(clips[1], rate, AudioFormat(24000)))
    assert torch.equal(torch.cat(codes), tok.encoder.forward(wav[None].to(DEV))[0].T.cpu())
    st.close()
    res.close()
    with pytest.raises(ValueError):
        tok.open_encode_stream(batch=1, sample_rate=12345)
