"""Scratch growth of the codec decoder, codec encoder and speaker encoder: a run of ever longer requests (the prefix
re-decode of TTSEngine.stream_synthesize(left_context=None), Qwen3TTSTokenizer.decode on longer and longer inputs) must
hold one scratch at a time.  An engine that grows its scratch frees the old block, so after the run this process's
device memory exceeds its level after the first call by no more than the scratch of the largest request.

Device memory is NVML's per-process figure (a read-only query): it sees the engines' cudaMalloc blocks, which the
torch allocator's counters do not.  What torch itself reserved over the run is subtracted."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MiB = 1 << 20
SLACK = 16 * MiB   # cudaMalloc rounds every block up to its 2 MiB pages


def _process_bytes():
    import pynvml
    p = torch.cuda.get_device_properties(0)
    pynvml.nvmlInit()
    try:
        h = pynvml.nvmlDeviceGetHandleByPciBusId(f"{p.pci_domain_id:08x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0")
        procs = pynvml.nvmlDeviceGetComputeRunningProcesses(h)
    finally:
        pynvml.nvmlShutdown()
    mine = [q for q in procs if q.pid == os.getpid()]
    # inside a PID namespace NVML reports pids this process cannot map; it holds a CUDA context, so a lone entry is it
    if not mine and len(procs) == 1:
        mine = procs
    if not mine or mine[0].usedGpuMemory is None:
        pytest.skip(f"NVML does not tell this process's device memory apart ({len(procs)} compute processes listed)")
    return mine[0].usedGpuMemory


def _growth(call, sizes):
    """Device memory added over calls 2..n, less what torch reserved over them."""
    call(sizes[0])
    torch.cuda.synchronize()
    m0, r0 = _process_bytes(), torch.cuda.memory_reserved()
    for s in sizes[1:]:
        call(s)
    torch.cuda.synchronize()
    return (_process_bytes() - m0) - (torch.cuda.memory_reserved() - r0)


def test_codec_decoder_scratch_does_not_accumulate():
    from oracle import codec as OC
    from qwen3_tts_b200.codec import CodecDecoder
    from tests.test_gpu_codec import _bf16_round, _pkg_cfg, _small_cfg
    cfg = _small_cfg()
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=5))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=64)
    g = torch.Generator().manual_seed(0)
    codes = torch.randint(0, cfg.codebook_size, (2, cfg.num_quantizers, 64), generator=g).to(DEV)
    # bf16 elements per (row, frame): the widest stage is the last decoder block, 1920 samples x 16 channels
    per_frame = 1920 * (cfg.decoder_dim >> len(cfg.upsample_rates))
    largest = 4 * 2 * per_frame * 2 * 64   # four buffers of B x T x per_frame bf16
    grown = _growth(lambda T: dec.forward(codes[..., :T]), list(range(4, 65, 4)))
    dec.close()
    assert grown <= largest + SLACK, f"{grown / MiB:.0f} MiB kept after growing requests (largest scratch {largest / MiB:.0f} MiB)"


def test_codec_encoder_scratch_does_not_accumulate():
    from oracle import mimi_encoder as M
    from qwen3_tts_b200.codec_encoder import CodecEncoder
    from tests.test_gpu_codec_encoder import _pkg_cfg
    cfg = M.cfg_tiny_encoder()
    enc = CodecEncoder(_pkg_cfg(cfg), M.random_weights(cfg, seed=3), device=DEV, max_frames=512)
    B, T = 2, 240000
    wav = (torch.randn(B, T, generator=torch.Generator().manual_seed(1)) * 0.1).clamp(-1, 1).to(DEV)
    # fp32 elements per (row, sample): the widest activation is conv0's num_filters channels at the full rate
    largest = 3 * 4 * cfg.num_filters * B * T   # three buffers
    grown = _growth(lambda n: enc.forward(wav[:, :n]), [24000 * i for i in range(1, 11)])
    assert grown <= largest + SLACK, f"{grown / MiB:.0f} MiB kept after growing requests (largest scratch {largest / MiB:.0f} MiB)"


def test_speaker_encoder_scratch_does_not_accumulate():
    from oracle import speaker_encoder as S
    from qwen3_tts_b200.speaker_encoder import SpeakerEncoder
    from tests.test_gpu_speaker_encoder import _pkg_cfg
    cfg = S.SpkEncCfg()
    enc = SpeakerEncoder(_pkg_cfg(cfg), S.random_weights(cfg, seed=1), device=DEV)
    B, T = 2, 192000
    wav = (torch.randn(B, T, generator=torch.Generator().manual_seed(2)) * 0.1).clamp(-1, 1).to(DEV)
    # fp32 elements per (row, frame): mel, block 0, 3 block-wide, 6 concatenation-wide and the attention channels
    C, Ccat = cfg.enc_channels[1], cfg.enc_channels[-1]
    per_frame = cfg.mel_dim + cfg.enc_channels[0] + 3 * C + 6 * Ccat + cfg.enc_attention_channels
    largest = 4 * B * (enc.frames(T) * per_frame + 2 * C + cfg.enc_se_channels + 2 * Ccat)
    grown = _growth(lambda n: enc.embed_waveform(wav[:, :n]), [24000 * i for i in range(1, 9)])
    assert grown <= largest + SLACK, f"{grown / MiB:.0f} MiB kept after growing requests (largest scratch {largest / MiB:.0f} MiB)"
