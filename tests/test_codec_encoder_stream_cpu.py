"""CPU side of the streaming codec encoder: the reference semantics it rests on (checked on the oracle, which
test_oracle_encoder.py pins to transformers' MimiModel), the framing arithmetic of EncoderStream.push / end, and the
argument checks that run before any native call."""
import numpy as np
import pytest
import torch

from oracle import mimi_encoder as M


def _wav(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(1, n, generator=g) * 0.1).clamp(-1, 1)


@pytest.mark.parametrize("which", ["tiny", "default"])
def test_whole_frame_prefix_codes_equal_the_full_clips(which):
    """Causality: the codes of a k-frame prefix are the first k frames of the whole clip's codes, so whole frames can
    be encoded as they arrive with carried state."""
    cfg = M.cfg_tiny_encoder() if which == "tiny" else M.MimiEncCfg()
    W = M.random_weights(cfg, seed=5)
    frames = 12 if which == "default" else 20
    wav = _wav(frames * cfg.hop + 700, 1)
    full = M.encode(W, cfg, wav)
    assert full.shape[2] == frames + 1
    for k in ((1, 5, frames) if which == "default" else (1, 3, 7, frames)):
        assert torch.equal(M.encode(W, cfg, wav[:, : k * cfg.hop]), full[:, :, :k]), k


def test_zero_padded_tail_is_not_the_clip_end():
    """The one-shot pads every layer on the right ("extra padding"), which differs from encoding zero audio: padding a
    clip to a whole number of frames changes its last frame.  So a stream encodes a clip's final partial frame on its
    own path instead of pushing zeros."""
    cfg = M.cfg_tiny_encoder()
    W = M.random_weights(cfg, seed=5)
    wav = _wav(4 * cfg.hop + 333, 2)
    clip = M.encode(W, cfg, wav)
    padded = M.encode(W, cfg, torch.cat([wav, torch.zeros(1, cfg.hop - 333)], 1))
    assert clip.shape == padded.shape
    assert torch.equal(clip[:, :, :4], padded[:, :, :4])
    assert not torch.equal(clip[:, :, 4], padded[:, :, 4])


def test_split_frames():
    from qwen3_tts_b200.codec_encoder import split_frames
    hop = 1920
    assert split_frames(0, 0, hop) == (0, 0)
    assert split_frames(0, 1919, hop) == (0, 1919)
    assert split_frames(1919, 1, hop) == (1, 0)
    assert split_frames(0, 1921, hop) == (1, 1)
    assert split_frames(1000, 9 * hop + 1000, hop) == (10, 80)
    # whatever the chunking, the frames sent plus what end() sends cover the clip exactly
    rng = np.random.default_rng(0)
    for _ in range(200):
        sizes = rng.integers(0, 3 * hop, size=int(rng.integers(1, 12)))
        held, sent = 0, 0
        for n in sizes:
            f, held = split_frames(held, int(n), hop)
            sent += f
            assert 0 <= held < hop
        assert sent * hop + held == int(sizes.sum())
        assert sent + (1 if held else 0) == -(-int(sizes.sum()) // hop)   # = the one-shot's frame count


def test_python_argument_checks():
    from qwen3_tts_b200.codec_encoder import check_chunks, check_rows
    ok = check_chunks({0: np.zeros(5, np.float64), 2: torch.ones(3)}, 3)
    assert ok[0].dtype == torch.float32 and ok[2].shape == (3,)
    for bad, what in (({3: np.zeros(4, np.float32)}, "row 3"), ({-1: np.zeros(4, np.float32)}, "row -1"),
                      ({0: np.zeros((2, 4), np.float32)}, "1-D"), ({1: np.array([1.0, np.inf], np.float32)}, "finite"),
                      ({0: torch.tensor([0.0, float("nan")])}, "finite"), ({0: np.zeros(3, np.int16)}, "floating"),
                      ({"0": np.zeros(3, np.float32)}, "row"), ([np.zeros(3, np.float32)], "dict")):
        with pytest.raises(ValueError, match=what):
            check_chunks(bad, 3)
    assert check_rows([2, 0], 3) == [2, 0] and check_rows(1, 3) == [1]
    for bad in ([3], [0, 0], [-1], [True]):
        with pytest.raises(ValueError):
            check_rows(bad, 3)
