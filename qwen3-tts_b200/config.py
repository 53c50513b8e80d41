"""Shape/config records for the hot path; every value is read from the loaded HF config objects
(never hard-coded: SURVEY §0 F6).  Mirrors core/models/configuration_qwen3_tts.py:187-212,370-404 and
core/tokenizer_12hz/configuration_qwen3_tts_tokenizer_v2.py:72-93 of the reference."""
import math
import numbers
import operator
from dataclasses import dataclass, field
from typing import Optional, Tuple


@dataclass
class StackConfig:
    hidden_size: int
    num_layers: int
    num_heads: int
    num_kv_heads: int
    head_dim: int
    intermediate_size: int
    vocab_size: int
    rms_eps: float = 1e-6
    rope_theta: float = 1e6


@dataclass
class TTSConfig:
    talker: StackConfig
    cp: StackConfig
    num_code_groups: int = 16
    text_hidden_size: int = 2048
    text_vocab_size: int = 151936
    codec_eos_token_id: int = 2150
    codec_pad_id: int = 2148
    codec_bos_id: int = 2149
    codec_think_id: int = 2154
    codec_nothink_id: int = 2155
    codec_think_bos_id: int = 2156
    codec_think_eos_id: int = 2157
    tts_bos_token_id: int = 151672
    tts_eos_token_id: int = 151673
    tts_pad_token_id: int = 151671

    @staticmethod
    def from_hf(cfg):
        """cfg: the reference's Qwen3TTSConfig (has .talker_config with .code_predictor_config)."""
        t = cfg.talker_config
        c = t.code_predictor_config

        def stack(s, theta_default):
            hd = getattr(s, "head_dim", None) or s.hidden_size // s.num_attention_heads
            return StackConfig(s.hidden_size, s.num_hidden_layers, s.num_attention_heads, s.num_key_value_heads, hd,
                               s.intermediate_size, s.vocab_size, float(s.rms_norm_eps),
                               float(getattr(s, "rope_theta", theta_default)))

        rs = getattr(t, "rope_scaling", None) or {}
        sec = rs.get("mrope_section")
        if sec is not None:
            hd = getattr(t, "head_dim", None) or t.hidden_size // t.num_attention_heads
            assert sum(sec) == hd // 2, "mrope sections must sum to head_dim/2"
        out = TTSConfig(talker=stack(t, 10000.0), cp=stack(c, 10000.0), num_code_groups=t.num_code_groups,
                        text_hidden_size=t.text_hidden_size, text_vocab_size=getattr(t, "text_vocab_size", 151936),
                        codec_eos_token_id=t.codec_eos_token_id, codec_pad_id=t.codec_pad_id,
                        codec_bos_id=t.codec_bos_id, codec_think_id=t.codec_think_id,
                        codec_nothink_id=t.codec_nothink_id, codec_think_bos_id=t.codec_think_bos_id,
                        codec_think_eos_id=t.codec_think_eos_id,
                        tts_bos_token_id=cfg.tts_bos_token_id, tts_eos_token_id=cfg.tts_eos_token_id,
                        tts_pad_token_id=cfg.tts_pad_token_id)
        V = out.talker.vocab_size
        assert V - 1024 <= out.codec_eos_token_id < V, "EOS must lie in the suppress range [V-1024, V)"
        return out


@dataclass
class SamplingParams:
    """inference/qwen3_tts_model.py:287-352 hard defaults."""
    do_sample: bool = True
    top_k: int = 50
    top_p: float = 1.0
    temperature: float = 0.9
    repetition_penalty: float = 1.05
    subtalker_dosample: bool = True
    subtalker_top_k: int = 50
    subtalker_top_p: float = 1.0
    subtalker_temperature: float = 0.9
    min_new_tokens: int = 2
    max_new_tokens: int = 2048
    suppress_eos: bool = False
    seed: int = 0


@dataclass
class CodecConfig:
    codebook_size: int = 2048
    codebook_dim: int = 512
    hidden_size: int = 1024
    latent_dim: int = 1024
    rope_theta: float = 10000.0
    num_heads: int = 16
    num_kv_heads: int = 16
    head_dim: int = 64
    sliding_window: int = 72
    intermediate_size: int = 3072
    rms_eps: float = 1e-5
    num_layers: int = 8
    num_quantizers: int = 16
    upsample_rates: Tuple[int, ...] = (8, 5, 4, 3)
    upsampling_ratios: Tuple[int, ...] = (2, 2)
    decoder_dim: int = 1536

    @property
    def total_upsample(self):
        n = 1
        for r in tuple(self.upsample_rates) + tuple(self.upsampling_ratios):
            n *= int(r)
        return n

    @staticmethod
    def from_hf(dc):
        hd = getattr(dc, "head_dim", None) or dc.hidden_size // dc.num_attention_heads
        return CodecConfig(dc.codebook_size, dc.codebook_dim, dc.hidden_size, dc.latent_dim, float(dc.rope_theta),
                           dc.num_attention_heads, dc.num_key_value_heads, hd, dc.sliding_window,
                           dc.intermediate_size, float(dc.rms_norm_eps), dc.num_hidden_layers, dc.num_quantizers,
                           tuple(dc.upsample_rates), tuple(dc.upsampling_ratios), dc.decoder_dim)


@dataclass
class EncoderConfig:
    """The codec ENCODER = transformers MimiConfig (the reference builds MimiConfig(**encoder_config),
    core/tokenizer_12hz/configuration_qwen3_tts_tokenizer_v2.py:155-162) + encoder_valid_num_quantizers (:147)."""
    num_filters: int = 64
    kernel_size: int = 7
    last_kernel_size: int = 3
    residual_kernel_size: int = 3
    compress: int = 2
    ratios: Tuple[int, ...] = (4, 5, 6, 8)      # encoder order = reversed(MimiConfig.upsampling_ratios)
    hidden_size: int = 512
    num_layers: int = 8
    num_heads: int = 8
    head_dim: int = 64
    intermediate_size: int = 2048
    sliding_window: int = 250
    rope_theta: float = 10000.0
    norm_eps: float = 1e-5
    codebook_size: int = 2048
    codebook_dim: int = 256
    num_semantic_quantizers: int = 1
    valid_num_quantizers: int = 16
    downsample_stride: int = 2
    max_position_embeddings: int = 8000
    encode_downsample_rate: int = 1920

    @staticmethod
    def from_hf(mc, valid_num_quantizers=16, encode_downsample_rate=1920):
        """mc: a transformers MimiConfig (Qwen3TTSTokenizerV2Config.encoder_config)."""
        rp = getattr(mc, "rope_parameters", None) or {}
        theta = rp.get("rope_theta") if isinstance(rp, dict) else None
        theta = theta or getattr(mc, "rope_theta", None) or 10000.0
        if getattr(mc, "num_residual_layers", 1) != 1 or getattr(mc, "use_conv_shortcut", False) or \
                not getattr(mc, "use_causal_conv", True) or mc.num_key_value_heads != mc.num_attention_heads:
            raise ValueError("unsupported MimiConfig variant (need 1 residual layer, identity shortcut, causal convs, MHA)")
        return EncoderConfig(mc.num_filters, mc.kernel_size, mc.last_kernel_size, mc.residual_kernel_size, mc.compress,
                             tuple(reversed(list(mc.upsampling_ratios))), mc.hidden_size, mc.num_hidden_layers,
                             mc.num_attention_heads, mc.head_dim, mc.intermediate_size, mc.sliding_window, float(theta),
                             float(mc.norm_eps), mc.codebook_size, mc.codebook_dim, mc.num_semantic_quantizers,
                             int(valid_num_quantizers), int(round(mc.encodec_frame_rate / mc.frame_rate)),
                             mc.max_position_embeddings, int(encode_downsample_rate))


@dataclass
class SpeakerEncoderConfig:
    """Qwen3TTSSpeakerEncoderConfig defaults (core/models/configuration_qwen3_tts.py:47-57) + the mel front-end constants
    hard-coded at the reference call site (modeling_qwen3_tts.py:1943-1951)."""
    mel_dim: int = 128
    enc_dim: int = 1024
    enc_channels: Tuple[int, ...] = (512, 512, 512, 512, 1536)
    enc_kernel_sizes: Tuple[int, ...] = (5, 3, 3, 3, 1)
    enc_dilations: Tuple[int, ...] = (1, 2, 3, 4, 1)
    enc_attention_channels: int = 128
    enc_res2net_scale: int = 8
    enc_se_channels: int = 128
    sample_rate: int = 24000
    n_fft: int = 1024
    hop_size: int = 256
    win_size: int = 1024
    fmin: float = 0.0
    fmax: float = 12000.0

    @staticmethod
    def from_dict(d):
        d = d or {}
        base = SpeakerEncoderConfig()
        kw = {k: (tuple(v) if isinstance(v, (list, tuple)) else v) for k, v in d.items() if hasattr(base, k)}
        return SpeakerEncoderConfig(**kw)


SUPPORTED_RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000)
ENCODINGS = ("f32", "s16", "ulaw")
SPEED_RANGE = (0.5, 2.0)
PITCH_RANGE = (-12.0, 12.0)    # semitones
VOLUME_RANGE = (-30.0, 12.0)   # dB
LOUDNESS_RANGE = (-40.0, -10.0)   # LUFS


def _real_in(name: str, v, lo: float, hi: float) -> float:
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)) or not lo <= float(v) <= hi:
        raise ValueError(f"{name} {v!r} is not a real number in [{lo}, {hi}]")
    return float(v)


@dataclass(frozen=True)
class AudioFormat:
    """The sample rate, encoding and prosody of a client's audio: "f32" float32 samples, "s16" 16-bit PCM (int16),
    "ulaw" 8-bit G.711 mu-law (uint8).  Rates: SUPPORTED_RATES.  `speed`: a real number in SPEED_RANGE, the pace of the
    speech (1.25 is 25 % faster, same pitch; audio.TimeStretch, resolution 1/480).  `pitch`: semitones in PITCH_RANGE
    (time-stretch, then rate conversion from 50*pitch_step Hz; formants move with it).  `volume`: dB in VOLUME_RANGE
    through audio.Limiter, peaks held at -1 dBFS.  `loudness`: None, or a target integrated loudness in LUFS in
    LOUDNESS_RANGE through audio.Loudness (BS.1770 gated loudness measured while the audio streams), always followed by
    the limiter at `volume`.  speed / (pitch_step/480) must lie in [0.5, 2] (hop in [240, 960]).  Anything else raises
    ValueError on construction."""
    sample_rate: int
    encoding: str = "f32"
    speed: float = 1.0
    pitch: float = 0.0
    volume: float = 0.0
    loudness: Optional[float] = None

    def __post_init__(self):
        try:
            sr = operator.index(self.sample_rate)   # int or numpy integer; not a float
        except TypeError:
            sr = None
        if sr is None or isinstance(self.sample_rate, bool) or sr not in SUPPORTED_RATES:
            raise ValueError(f"sample_rate {self.sample_rate!r} is not supported; supported rates: {SUPPORTED_RATES}")
        if not isinstance(self.encoding, str) or self.encoding not in ENCODINGS:
            raise ValueError(f"encoding {self.encoding!r} is not supported; supported encodings: {ENCODINGS}")
        object.__setattr__(self, "sample_rate", sr)
        object.__setattr__(self, "speed", _real_in("speed", self.speed, *SPEED_RANGE))
        object.__setattr__(self, "pitch", _real_in("pitch", self.pitch, *PITCH_RANGE))
        object.__setattr__(self, "volume", _real_in("volume", self.volume, *VOLUME_RANGE))
        if self.loudness is not None:
            object.__setattr__(self, "loudness", _real_in("loudness", self.loudness, *LOUDNESS_RANGE))
        if not 240 <= self.hop <= 960:
            raise ValueError(f"speed {self.speed} at pitch {self.pitch} gives a time-stretch hop of {self.hop}: speed "
                             f"divided by the pitch factor {self.pitch_step}/480 must lie in [0.5, 2]")

    @property
    def pitch_step(self) -> int:
        """Lp = floor(480 * 2^(pitch/12) + 0.5), in [240, 960]: the pitch factor is Lp/480."""
        return int(math.floor(480 * 2.0 ** (self.pitch / 12) + 0.5))

    @property
    def hop(self) -> int:
        """The time-stretch's analysis hop Ha = floor(speed * 480 * (480/Lp) + 0.5) (floor(speed*480 + 0.5) at pitch 0);
        the effective speed is Ha*Lp/480^2."""
        return int(math.floor(self.speed * 480 * (480 / self.pitch_step) + 0.5))
