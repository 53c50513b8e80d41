"""Host-side mirror of the reference's Python API on top of the H100 engines (drop-in boundary, SURVEY §8b).

  * `Qwen3TTSForConditionalGenerationB200.generate(...)`  == core/models/modeling_qwen3_tts.py:2022-2292 (a1): builds the
    per-sample prefill embeddings exactly as the reference does (role / think-language-speaker prefix / text / ICL,
    SURVEY App. A.1) with plain PyTorch ops, then hands them to the fused AR engine (seam B) instead of
    `talker.generate`, and returns the per-sample code lists trimmed at the first EOS.
  * `Qwen3TTSModel`      == inference/qwen3_tts_model.py:54 (generate_custom_voice / voice_design / voice_clone).
  * `Qwen3TTSTokenizer`  == inference/qwen3_tts_tokenizer.py:44 (encode() on the fp32 codec encoder, decode()).

Construction takes a state_dict + config + a `processor` callable (`processor(text=..., return_tensors="pt")
["input_ids"]`); `from_pretrained` (checkpoint.py) builds those from a HF checkpoint directory like the reference's.
"""
from dataclasses import dataclass
import dataclasses
import os
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F

from .codec import CodecDecoder
from .config import CodecConfig, SamplingParams, TTSConfig
from .engine import AREngine


@dataclass
class VoiceClonePromptItem:
    """inference/qwen3_tts_model.py:40-51."""
    ref_code: Optional[torch.Tensor]
    ref_spk_embedding: torch.Tensor
    x_vector_only_mode: bool
    icl_mode: bool
    ref_text: Optional[str] = None


class Voice:
    """A registered voice (Qwen3TTSModel.register_voice): `prefix`, the (P, H) prompt rows every request of the voice
    begins with, whose talker K/V live in the AR engine as prefix `prefix_id`; for an ICL clone, the codec decoder's
    state after its reference codes in row `bank` = (bank, row) of the decoder's reference bank.  `pending` counts its
    requests a batcher has queued but not admitted; running requests hold their own copies."""

    def __init__(self, owner, language, speaker, instruct_ids, vcp, ref_ids, non_streaming_mode, icl):
        self.engine = owner.model.engine
        self.language, self.speaker, self.instruct_ids = language, speaker, instruct_ids
        self.vcp, self.ref_ids, self.non_streaming_mode, self.icl = vcp, ref_ids, non_streaming_mode, icl
        self.prefix: Optional[torch.Tensor] = None
        self.prefix_id: Optional[int] = None
        self.codec = None
        self.ref_codes: Optional[torch.Tensor] = None
        self.bank: Optional[Tuple[int, int]] = None
        self.pending = 0
        self.closed = False

    @property
    def prefix_len(self) -> int:
        return int(self.prefix.shape[0])

    @property
    def ref_len(self) -> int:
        """Frames of the reference the voice's audio continues (0 without one)."""
        return 0 if self.ref_codes is None else int(self.ref_codes.shape[0])

    def close(self):
        """Free the voice's prefix and reference-bank row.  ValueError while a batcher holds pending requests of it."""
        if self.closed:
            return
        if self.pending:
            raise ValueError(f"the voice has {self.pending} pending requests")
        self.engine.free_prefix(self.prefix_id)
        if self.bank is not None:
            self.codec.bank_release(*self.bank)
        self.closed = True


class Qwen3TTSForConditionalGenerationB200:
    def __init__(self, cfg: TTSConfig, weights: Dict[str, torch.Tensor], device="cuda:0", spk_id=None,
                 spk_is_dialect=None, codec_language_id=None, tts_model_type="custom_voice", tts_model_size="1b7",
                 max_batch=32, max_ctx=4096, engine: Optional[AREngine] = None):
        self.cfg = cfg
        self.device = torch.device(device)
        self.dtype = torch.bfloat16
        self.spk_id = {k.lower(): v for k, v in (spk_id or {}).items()}
        self.spk_is_dialect = {k.lower(): v for k, v in (spk_is_dialect or {}).items()}
        self.codec_language_id = {k.lower(): v for k, v in (codec_language_id or {}).items()}
        self.tts_model_type, self.tts_model_size = tts_model_type, tts_model_size
        g = lambda n: weights[n].detach().to(self.device, self.dtype)  # noqa: E731
        self.text_embedding = g("talker.model.text_embedding.weight")
        self.fc1_w, self.fc1_b = g("talker.text_projection.linear_fc1.weight"), g("talker.text_projection.linear_fc1.bias")
        self.fc2_w, self.fc2_b = g("talker.text_projection.linear_fc2.weight"), g("talker.text_projection.linear_fc2.bias")
        self.codec_embedding = g("talker.model.codec_embedding.weight")
        self.cp_embeddings = [g(f"talker.code_predictor.model.codec_embedding.{j}.weight")
                              for j in range(cfg.num_code_groups - 1)]
        self.engine = engine or AREngine(cfg, weights, device=device, max_batch=max_batch, max_ctx=max_ctx)
        self.speech_tokenizer = None
        self.speaker_encoder = None            # SpeakerEncoder (Base checkpoints), see load_speaker_encoder
        self.speaker_encoder_sample_rate = 24000
        self.tokenizer_type = None
        self.generate_config = None
        self.supported_speakers = self.spk_id.keys()
        self.supported_languages = ["auto"] + [k for k in self.codec_language_id if "dialect" not in k]

    # -- small helpers restating the reference's embedding calls
    def _tp(self, ids: torch.Tensor) -> torch.Tensor:
        """text_projection(text_embedding(ids)) — ResizeMLP: Linear(bias) -> SiLU -> Linear(bias) (:808-816)."""
        x = F.embedding(ids.to(self.device), self.text_embedding)
        return F.linear(F.silu(F.linear(x, self.fc1_w, self.fc1_b)), self.fc2_w, self.fc2_b)

    def _ce(self, ids) -> torch.Tensor:
        return F.embedding(torch.as_tensor(ids, device=self.device, dtype=torch.long), self.codec_embedding)

    def load_speech_tokenizer(self, speech_tokenizer):
        self.speech_tokenizer = speech_tokenizer

    def load_generate_config(self, generate_config):
        self.generate_config = generate_config

    def load_speaker_encoder(self, speaker_encoder):
        self.speaker_encoder = speaker_encoder
        self.speaker_encoder_sample_rate = int(speaker_encoder.cfg.sample_rate)

    def extract_speaker_embedding(self, audio: np.ndarray, sr: int) -> torch.Tensor:
        """:1941-1954 — 24 kHz mono waveform -> (enc_dim,) x-vector in the model dtype."""
        assert sr == 24000, "Only support 24kHz audio"
        if self.speaker_encoder is None:
            raise RuntimeError("this model was built without speaker-encoder weights (only Base checkpoints carry them)")
        emb = self.speaker_encoder.embed_waveform(torch.from_numpy(np.ascontiguousarray(audio, dtype=np.float32))[None])[0]
        return emb.to(self.dtype)

    def get_supported_speakers(self):
        return self.supported_speakers

    def get_supported_languages(self):
        return self.supported_languages

    def generate_icl_prompt(self, text_id, ref_id, ref_code, tts_pad_embed, tts_eos_embed, non_streaming_mode):
        """:1968-2019."""
        text_embed = self._tp(torch.cat([ref_id, text_id], dim=-1))
        text_embed = torch.cat([text_embed, tts_eos_embed], dim=1)
        ref_code = ref_code.to(self.device)
        parts = [F.embedding(ref_code[:, :1], self.codec_embedding)]
        for i in range(1, self.cfg.num_code_groups):
            parts.append(F.embedding(ref_code[:, i:i + 1], self.cp_embeddings[i - 1]))
        codec_embed = torch.cat(parts, dim=1).sum(1).unsqueeze(0)
        codec_embed = torch.cat([self._ce([[self.cfg.codec_bos_id]]), codec_embed], dim=1)
        text_lens, codec_lens = text_embed.shape[1], codec_embed.shape[1]
        if non_streaming_mode:
            icl = text_embed + self._ce([[self.cfg.codec_pad_id] * text_lens])
            icl = torch.cat([icl, codec_embed + tts_pad_embed], dim=1)
            return icl, tts_pad_embed
        if text_lens > codec_lens:
            return text_embed[:, :codec_lens] + codec_embed, text_embed[:, codec_lens:]
        text_embed = torch.cat([text_embed] + [tts_pad_embed] * (codec_lens - text_lens), dim=1)
        return text_embed + codec_embed, tts_pad_embed

    # ------------------------------------------------------------------ batched prefill assembly (SURVEY §8f-3)
    def _plan_sample(self, input_id, instruct, ref_id, vcp, index, language, speaker, non_streaming_mode, live=False):
        """Index plan of one sample (:2086-2234): every prefill / trailing position is `TP(text id) + codec source`
        with either side optional.  Returns (text_ids, codec_src, trailing_ids); text id -1 = no text part; codec_src
        entries: None | ("ce", id) | ("spk",) | ("icl", frame).  `live` (streaming ICL layout only): the ids are the
        text known so far, the text stream has no tts_eos yet, and the ICL positions its text has not reached carry their
        codec part alone (text id -1)."""
        cfg = self.cfg
        ids = [int(x) for x in input_id.reshape(-1).tolist()]
        BOS, EOS, PAD = cfg.tts_bos_token_id, cfg.tts_eos_token_id, cfg.tts_pad_token_id
        has_spk_vec = False
        speaker_id = None
        if vcp is None:
            if not (speaker == "" or speaker is None):
                if speaker.lower() not in self.spk_id:
                    raise NotImplementedError(f"Speaker {speaker} not implemented")
                speaker_id = self.spk_id[speaker.lower()]
        else:
            has_spk_vec = bool(vcp["x_vector_only_mode"][index] or vcp["icl_mode"][index])
        assert language is not None
        if language.lower() == "auto":
            language_id = None
        else:
            if language.lower() not in self.codec_language_id:
                raise NotImplementedError(f"Language {language} not implemented")
            language_id = self.codec_language_id[language.lower()]
        if (language.lower() in ["chinese", "auto"] and speaker != "" and speaker is not None
                and self.spk_is_dialect.get(speaker.lower(), False) is not False):
            language_id = self.codec_language_id[self.spk_is_dialect[speaker.lower()]]
        if language_id is None:
            cids = [cfg.codec_nothink_id, cfg.codec_think_bos_id, cfg.codec_think_eos_id]
        else:
            cids = [cfg.codec_think_id, cfg.codec_think_bos_id, language_id, cfg.codec_think_eos_id]
        C = [("ce", c) for c in cids]
        if has_spk_vec:
            C.append(("spk",))
        elif speaker_id is not None:
            C.append(("ce", speaker_id))
        C += [("ce", cfg.codec_pad_id), ("ce", cfg.codec_bos_id)]
        text, codec = [], []
        if instruct is not None:
            for t in instruct.reshape(-1).tolist():
                text.append(int(t)); codec.append(None)
        for t in ids[:3]:                                    # role tokens (:2177-2179)
            text.append(t); codec.append(None)
        n_over = len(C) - 1                                  # overlay (:2182-2184)
        text += [PAD] * (n_over - 1) + [BOS]
        codec += C[:-1]
        icl = vcp is not None and vcp["ref_code"] is not None and vcp["icl_mode"][index]
        if icl:                                              # generate_icl_prompt (:1968-2019)
            rid = [int(x) for x in ref_id.reshape(-1).tolist()][3:-2]
            tstream = rid + ids[3:-5] + ([] if live else [EOS])
            n_ref = int(vcp["ref_code"][index].shape[0])
            cstream = [("ce", cfg.codec_bos_id)] + [("icl", t) for t in range(n_ref)]
            Lt, Lc = len(tstream), len(cstream)
            if live:
                text += tstream[:Lc] + [-1] * (Lc - min(Lt, Lc)); codec += cstream
                trailing = tstream[Lc:]
            elif non_streaming_mode:
                text += tstream + [PAD] * Lc
                codec += [("ce", cfg.codec_pad_id)] * Lt + cstream
                trailing = [PAD]
            elif Lt > Lc:
                text += tstream[:Lc]; codec += cstream
                trailing = tstream[Lc:]
            else:
                text += tstream + [PAD] * (Lc - Lt); codec += cstream
                trailing = [PAD]
        elif non_streaming_mode:                             # (:2203-2227)
            body = ids[3:-5]
            text += body + [EOS] + [PAD]
            codec += [("ce", cfg.codec_pad_id)] * (len(body) + 1) + [("ce", cfg.codec_bos_id)]
            trailing = [PAD]
        else:                                                # (:2199-2202, :2229-2232)
            text.append(ids[3]); codec.append(C[-1])
            trailing = ids[4:-5] + [EOS]
        return text, codec, trailing

    @torch.no_grad()
    def build_prefill(self, input_ids, instruct_ids=None, ref_ids=None, voice_clone_prompt=None, languages=None,
                      speakers=None, non_streaming_mode=False):
        """:2068-2237 — per-sample (unpadded) prefill embeddings + trailing text + tts_pad, computed for the WHOLE request
        list with a fixed number of batched device launches (one text-embedding gather + one ResizeMLP over every text
        token of every sample, one codec-embedding gather, one 16-codebook gather-and-sum over all ICL reference
        frames, one add) instead of dozens of small launches per sample.  The index plan is host-side integer work;
        `build_prefill_per_sample` is the statement-by-statement restatement it must equal.  The reference's left
        padding / attention mask (:2239-2254) is not materialised: the engine takes per-sequence lengths."""
        n = len(input_ids)
        if speakers is None:
            speakers = [None] * n
        plans = []
        for i in range(n):
            ins = instruct_ids[i] if instruct_ids is not None else None
            rid = ref_ids[i] if ref_ids is not None else None
            plans.append(self._plan_sample(input_ids[i], ins, rid, voice_clone_prompt, i, languages[i], speakers[i], non_streaming_mode))
        return self._embed_plans(plans, voice_clone_prompt)

    def _embed_plans(self, plans, voice_clone_prompt):
        """The rows of index plans (_plan_sample) with build_prefill's batched launches: (per-sample prompt rows,
        per-sample trailing rows, tts_pad_embed)."""
        cfg, dev = self.cfg, self.device
        H = self.codec_embedding.shape[1]
        # ---- text side: every text id of every sample (prefill + trailing) + the three specials, ONE ResizeMLP
        flat_text, seg = [], []
        for text, _, trailing in plans:
            seg.append((len(flat_text), len(text), len(trailing)))
            flat_text += [t if t >= 0 else cfg.tts_pad_token_id for t in text] + trailing
        flat_text += [cfg.tts_bos_token_id, cfg.tts_eos_token_id, cfg.tts_pad_token_id]
        tp = self._tp(torch.tensor(flat_text, dtype=torch.long, device=dev)[None])[0]          # (Ntext, H)
        tts_pad_embed = tp[-1]
        # ---- codec side: gather ids, speaker vectors, ICL frame sums
        ce_ids, ce_pos, spk_pos, icl_pos, icl_rows = [], [], [], [], []
        total = 0
        offs = []
        for i, (text, codec, _) in enumerate(plans):
            offs.append(total)
            for p, c in enumerate(codec):
                if c is None:
                    continue
                if c[0] == "ce":
                    ce_ids.append(c[1]); ce_pos.append(total + p)
                elif c[0] == "spk":
                    spk_pos.append((total + p, i))
                else:
                    icl_pos.append(total + p); icl_rows.append((i, c[1]))
            total += len(text)
        cpart = torch.zeros(total, H, dtype=self.dtype, device=dev)
        if ce_ids:
            cpart[torch.tensor(ce_pos, device=dev)] = F.embedding(torch.tensor(ce_ids, dtype=torch.long, device=dev), self.codec_embedding)
        for pos, i in spk_pos:
            cpart[pos] = voice_clone_prompt["ref_spk_embedding"][i].to(dev).to(self.dtype).reshape(-1)
        if icl_rows:
            G = cfg.num_code_groups
            ref = torch.stack([voice_clone_prompt["ref_code"][i][t].to(dev) for i, t in icl_rows])       # (R, G)
            parts = [F.embedding(ref[:, :1], self.codec_embedding)]
            for g in range(1, G):
                parts.append(F.embedding(ref[:, g:g + 1], self.cp_embeddings[g - 1]))
            cpart[torch.tensor(icl_pos, device=dev)] = torch.cat(parts, dim=1).sum(1)                    # == :1983-1998
        # ---- assemble: position = text part + codec part (either may be absent)
        embeds, trailing = [], []
        for i, (text, codec, trail) in enumerate(plans):
            t0, nt, ntr = seg[i]
            tpart = tp[t0:t0 + nt]
            has_text = torch.tensor([t >= 0 for t in text], device=dev)
            has_codec = torch.tensor([c is not None for c in codec], device=dev)
            cp_i = cpart[offs[i]:offs[i] + nt]
            both = tpart + cp_i
            emb = torch.where((has_text & has_codec)[:, None], both, torch.where(has_text[:, None], tpart, cp_i))
            embeds.append(emb)
            trailing.append(tp[t0 + nt:t0 + nt + ntr])
        return embeds, trailing, tts_pad_embed.reshape(-1)

    @torch.no_grad()
    def build_live_prefill(self, input_ids, instruct_ids=None, voice_clone_prompt=None, languages=None, speakers=None):
        """Live text: the streaming-layout prefill (build_prefill with non_streaming_mode=False, :2199-2202 / :2229-2232)
        of the text known so far.  The prefill holds the first text token; the trailing rows are the rest of the ids
        (`ids[4:-5]`) WITHOUT the final tts_eos row, which is appended (tts_eos_row) when the text ends.  A request
        whose later ids arrive through text_rows() and end with tts_eos_row() has exactly the prefill and trailing rows
        of build_prefill(non_streaming_mode=False) over all its ids.  ICL voice-clone prompts are refused: their prefill
        consumes the target text.  A text without tokens yet is refused too."""
        vcp = voice_clone_prompt
        for i, ids in enumerate(input_ids):
            if int(ids.reshape(-1).shape[0]) < 9:   # 3 role tokens, >= 1 text token, 5 closing tokens
                raise ValueError(f"request {i}: live text needs at least one text token in the prefill")
            if vcp is not None and vcp["ref_code"] is not None and vcp["icl_mode"][i]:
                raise ValueError(f"request {i}: an ICL voice-clone prompt cannot take live text here (its prefill consumes "
                                 f"the target text); use build_live_icl_prefill")
        embeds, trailing, pad = self.build_prefill(input_ids, instruct_ids, None, vcp, languages, speakers, non_streaming_mode=False)
        return embeds, [t[:-1] for t in trailing], pad

    @torch.no_grad()
    def build_live_icl_prefill(self, input_ids, ref_ids, voice_clone_prompt, languages):
        """Live text for ICL voice-clone prompts in the streaming layout (:1968-2019): (inputs_embeds, trailing,
        tts_pad_embed, overlay), lists per sample but the pad.  The ICL block's position j sums the text stream
        (reference text R tokens, target text, tts_eos) and the codec stream (codec_bos, the reference's frames: Lc =
        1 + frames), so its last K = max(0, Lc - R) positions each wait for one row of target text.  `inputs_embeds`
        are the prompt rows complete with the text known so far (the first min(K, T) target tokens summed onto their
        reference rows), `overlay` the (K - min(K, T), H) codec parts of the positions still waiting, in order, and
        `trailing` the known text rows past the ICL block, without tts_eos.  The text's later rows (text_rows, then
        tts_eos_row) complete the overlay first (overlay[i] + row) and then continue the trailing rows; if the text ends
        first, the rest of the overlay takes tts_pad_embed and the trailing rows are [tts_pad].  The rows are then
        exactly those of build_prefill(non_streaming_mode=False) over all the ids.  A text without tokens is accepted;
        every prompt must be an ICL one (the others take build_live_prefill)."""
        vcp = voice_clone_prompt
        for i in range(len(input_ids)):
            if vcp is None or vcp["ref_code"] is None or vcp["ref_code"][i] is None or not vcp["icl_mode"][i]:
                raise ValueError(f"request {i}: not an ICL voice-clone prompt; live text of other prompts takes "
                                 f"build_live_prefill")
            if int(input_ids[i].reshape(-1).shape[0]) < 8:   # 3 role tokens, 5 closing tokens
                raise ValueError(f"request {i}: the ids lack the chat wrapper's 3 role and 5 closing tokens")
        plans = [self._plan_sample(input_ids[i], None, ref_ids[i], vcp, i, languages[i], None, False, live=True)
                 for i in range(len(input_ids))]
        embeds, trailing, pad = self._embed_plans(plans, vcp)
        n_over = [sum(t < 0 for t in text[-int(vcp["ref_code"][i].shape[0]) - 1:]) for i, (text, _, _) in enumerate(plans)]
        return [e[:e.shape[0] - k] for e, k in zip(embeds, n_over)], trailing, pad, [e[e.shape[0] - k:] for e, k in zip(embeds, n_over)]

    @torch.no_grad()
    def text_rows(self, ids) -> torch.Tensor:
        """Trailing rows (n, H) of n more text ids of a live request: text_projection(text_embedding(ids))."""
        return self._tp(torch.as_tensor(ids, dtype=torch.long).reshape(1, -1))[0]

    @torch.no_grad()
    def tts_eos_row(self) -> torch.Tensor:
        """The (1, H) trailing row that ends a live request's text (the last trailing row of the streaming layout)."""
        return self.text_rows([self.cfg.tts_eos_token_id])

    @torch.no_grad()
    def build_prefill_per_sample(self, input_ids, instruct_ids=None, ref_ids=None, voice_clone_prompt=None, languages=None,
                      speakers=None, non_streaming_mode=False):
        """:2068-2237 restated statement by statement (one small embedding / MLP launch per piece and per sample, as
        the reference does).  Kept as the readable specification of `build_prefill`, which computes the same tensors
        with a handful of batched launches; tests/test_wrappers_cpu.py requires the two to agree exactly."""
        cfg = self.cfg
        n = len(input_ids)
        pieces: List[List[torch.Tensor]] = [[] for _ in range(n)]
        spk_embeds = None
        if voice_clone_prompt is not None:
            spk_embeds = [e.to(self.device).to(self.dtype) for e in voice_clone_prompt["ref_spk_embedding"]]
        if instruct_ids is not None:
            for i, ins in enumerate(instruct_ids):
                if ins is not None:
                    pieces[i].append(self._tp(ins))
        trailing = []
        if speakers is None:
            speakers = [None] * n
        tts_pad_embed = None
        for index, (input_id, language, speaker) in enumerate(zip(input_ids, languages, speakers)):
            input_id = input_id.to(self.device)
            if spk_embeds is None:
                if speaker == "" or speaker is None:
                    speaker_embed = None
                else:
                    if speaker.lower() not in self.spk_id:
                        raise NotImplementedError(f"Speaker {speaker} not implemented")
                    speaker_embed = self._ce(self.spk_id[speaker.lower()])
            else:
                if voice_clone_prompt["x_vector_only_mode"][index] or voice_clone_prompt["icl_mode"][index]:
                    speaker_embed = spk_embeds[index]
                else:
                    speaker_embed = None
            assert language is not None
            if language.lower() == "auto":
                language_id = None
            else:
                if language.lower() not in self.codec_language_id:
                    raise NotImplementedError(f"Language {language} not implemented")
                language_id = self.codec_language_id[language.lower()]
            if (language.lower() in ["chinese", "auto"] and speaker != "" and speaker is not None
                    and self.spk_is_dialect.get(speaker.lower(), False) is not False):
                language_id = self.codec_language_id[self.spk_is_dialect[speaker.lower()]]
            tts_bos_embed, tts_eos_embed, tts_pad_embed = self._tp(torch.tensor(
                [[cfg.tts_bos_token_id, cfg.tts_eos_token_id, cfg.tts_pad_token_id]], device=self.device)).chunk(3, dim=1)
            if language_id is None:
                prefill = [[cfg.codec_nothink_id, cfg.codec_think_bos_id, cfg.codec_think_eos_id]]
            else:
                prefill = [[cfg.codec_think_id, cfg.codec_think_bos_id, language_id, cfg.codec_think_eos_id]]
            e0 = self._ce(prefill)
            e1 = self._ce([[cfg.codec_pad_id, cfg.codec_bos_id]])
            if speaker_embed is None:
                codec_in = torch.cat([e0, e1], dim=1)
            else:
                codec_in = torch.cat([e0, speaker_embed.view(1, 1, -1), e1], dim=1)
            role = self._tp(input_id[:, :3])
            overlay = torch.cat((tts_pad_embed.expand(-1, codec_in.shape[1] - 2, -1), tts_bos_embed), dim=1) + codec_in[:, :-1]
            emb = torch.cat((role, overlay), dim=1)
            if (voice_clone_prompt is not None and voice_clone_prompt["ref_code"] is not None
                    and voice_clone_prompt["icl_mode"][index]):
                icl, trail = self.generate_icl_prompt(input_id[:, 3:-5], ref_ids[index][:, 3:-2].to(self.device),
                                                      voice_clone_prompt["ref_code"][index], tts_pad_embed, tts_eos_embed,
                                                      non_streaming_mode)
                emb = torch.cat([emb, icl], dim=1)
            else:
                emb = torch.cat([emb, self._tp(input_id[:, 3:4]) + codec_in[:, -1:]], dim=1)
                if non_streaming_mode:
                    emb = emb[:, :-1]
                    T = input_id[:, 3:-5].shape[1]
                    emb = torch.cat([emb,
                                     torch.cat((self._tp(input_id[:, 3:-5]), tts_eos_embed), dim=1)
                                     + self._ce([[cfg.codec_pad_id] * (T + 1)]),
                                     tts_pad_embed + self._ce([[cfg.codec_bos_id]])], dim=1)
                    trail = tts_pad_embed
                else:
                    trail = torch.cat((self._tp(input_id[:, 4:-5]), tts_eos_embed), dim=1)
            pieces[index].append(emb)
            trailing.append(trail)
        embeds = [torch.cat(p, dim=1).squeeze(0) for p in pieces]
        trailing = [t.squeeze(0) for t in trailing]
        return embeds, trailing, tts_pad_embed.reshape(-1)

    @torch.no_grad()
    def generate(self, input_ids=None, instruct_ids=None, ref_ids=None, voice_clone_prompt=None, languages=None,
                 speakers=None, non_streaming_mode=False, max_new_tokens: int = 4096, do_sample: bool = True,
                 top_k: int = 50, top_p: float = 1.0, temperature: float = 0.9, subtalker_dosample: bool = True,
                 subtalker_top_k: int = 50, subtalker_top_p: float = 1.0, subtalker_temperature: float = 0.9,
                 eos_token_id: Optional[int] = None, repetition_penalty: float = 1.05, seed: Optional[int] = None, **kwargs):
        """Signature and return of :2022-2043 / :2292: (codes list, per-step hidden-state list).  The reference's own
        wrappers discard the second value (SURVEY App. B.3); it is captured by the head phase of the fused kernel."""
        embeds, trailing, pad = self.build_prefill(input_ids, instruct_ids, ref_ids, voice_clone_prompt, languages,
                                                   speakers, non_streaming_mode)
        if eos_token_id is not None and eos_token_id != self.cfg.codec_eos_token_id:
            raise ValueError("eos_token_id must equal config.talker_config.codec_eos_token_id in the fused engine")
        if seed is None:
            # the reference samples from torch's global RNG (torch.multinomial): repeated calls differ and
            # torch.manual_seed() makes them reproducible — draw the Philox key from that same generator
            seed = int(torch.randint(0, 2 ** 62, (), dtype=torch.int64).item())
        sp = SamplingParams(do_sample=do_sample, top_k=top_k, top_p=top_p, temperature=temperature,
                            repetition_penalty=repetition_penalty, subtalker_dosample=subtalker_dosample,
                            subtalker_top_k=subtalker_top_k, subtalker_top_p=subtalker_top_p,
                            subtalker_temperature=subtalker_temperature, min_new_tokens=2, max_new_tokens=max_new_tokens,
                            seed=seed)
        tr = trailing
        out: List[torch.Tensor] = []
        hids: List[torch.Tensor] = []
        mb = self.engine.max_batch
        for s in range(0, len(embeds), mb):  # the reference runs one padded batch; we tile by engine capacity
            # Philox streams are keyed (seed; row, frame, group) with the row index local to a tile: give every
            # tile its own key so row b of two tiles never shares uniforms
            sp_t = sp if s == 0 else dataclasses.replace(sp, seed=(sp.seed ^ (s * 0x9E3779B97F4A7C15)) & (2 ** 63 - 1))
            c, h = self.engine.generate(embeds[s:s + mb], tr[s:s + mb], pad, sp_t, return_hidden=True)
            out += c
            hids += h
        return out, hids


# ----------------------------------------------------------------------------------------------------------------
class Qwen3TTSTokenizer:
    """inference/qwen3_tts_tokenizer.py:44 — decode path on the H100 codec engine."""

    def __init__(self, cfg: CodecConfig, weights, device="cuda:0", max_frames=1024, encoder_cfg=None,
                 encoder_weights=None):
        """`encoder_cfg` / `encoder_weights` (EncoderConfig + MimiModel-named state dict) enable encode(); without
        them the wrapper is decode-only (what TTS generation needs)."""
        self.config = cfg
        self.device = torch.device(device)
        self.decoder = CodecDecoder(cfg, weights, device=device, max_frames=max_frames)
        self.encoder = None
        if encoder_cfg is not None:
            from .codec_encoder import CodecEncoder
            self.encoder = CodecEncoder(encoder_cfg, encoder_weights, device=device)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, device_map="cuda:0", max_frames=1024,
                        with_encoder=True, **kwargs) -> "Qwen3TTSTokenizer":
        """inference/qwen3_tts_tokenizer.py:63-99 — a local HF directory (config.json + safetensors of
        Qwen3TTSTokenizerV2Model).  `device_map` names the CUDA device; `dtype` / `attn_implementation` kwargs of the
        reference are accepted; the engines fix their own precisions (bf16 tensor-core decoder, fp32 encoder) and a request
        for an fp32 decoder is answered with a RuntimeWarning rather than silently narrowed."""
        from . import checkpoint
        want = kwargs.get("dtype", kwargs.get("torch_dtype"))
        if want is not None and str(want).replace("torch.", "") in ("float32", "float", "float64", "double"):
            # not silent: the reference's standalone tokenizer (examples/test_tokenizer_12hz.py) runs in fp32
            import warnings
            warnings.warn(f"Qwen3TTSTokenizer: dtype={want} requested, but the H100 codec DECODER always computes in bf16 on the "
                          "tensor cores (fp32 accumulation; ~30 dB SNR against an fp32 forward, DESIGN.md section 5); the "
                          "ENCODER runs in fp32 and returns the same codes as the fp32 reference.", RuntimeWarning, stacklevel=2)
        d = checkpoint.resolve_dir(pretrained_model_name_or_path)
        cfg_json = checkpoint.read_json(os.path.join(d, "config.json"))
        mt = cfg_json.get("model_type", "qwen3_tts_tokenizer_12hz")
        if mt != "qwen3_tts_tokenizer_12hz":
            raise ValueError(f"unsupported tokenizer model_type {mt!r} (only the 12 Hz tokenizer is built)")
        device = device_map if isinstance(device_map, (str, torch.device)) else "cuda:0"
        ccfg, dec, ecfg, enc, rates = checkpoint.load_speech_tokenizer_checkpoint(d, device=device)
        use_enc = with_encoder and len(enc) > 0
        inst = cls(ccfg, dec, device=device, max_frames=max_frames, encoder_cfg=ecfg if use_enc else None,
                   encoder_weights=enc if use_enc else None)
        inst.rates = rates
        return inst

    rates = dict(input_sample_rate=24000, output_sample_rate=24000, decode_upsample_rate=None, encode_downsample_rate=None)

    def get_model_type(self):
        return "qwen3_tts_tokenizer_12hz"

    def get_input_sample_rate(self):
        return int(self.rates["input_sample_rate"])

    def get_output_sample_rate(self):
        return int(self.rates["output_sample_rate"])

    def get_encode_downsample_rate(self):
        return int(self.rates["encode_downsample_rate"] or self.config.total_upsample)

    def get_decode_upsample_rate(self):
        return int(self.rates["decode_upsample_rate"] or self.config.total_upsample)

    # ---- audio input normalisation (inference/qwen3_tts_tokenizer.py:100-207), host-only
    @staticmethod
    def _is_probably_base64(s: str) -> bool:
        return s.startswith("data:audio") or (("/" not in s and "\\" not in s) and len(s) > 256)

    @staticmethod
    def _is_url(s: str) -> bool:
        from urllib.parse import urlparse
        try:
            u = urlparse(s)
            return u.scheme in ("http", "https") and bool(u.netloc)
        except Exception:
            return False

    @staticmethod
    def _resample(a: np.ndarray, sr: int, target_sr: int) -> np.ndarray:
        """The reference calls librosa.resample (soxr); neither is in this image, so a polyphase FIR resampler
        (scipy.signal.resample_poly) stands in — same rate change, not bit-identical samples."""
        if int(sr) == int(target_sr):
            return a.astype(np.float32)
        from math import gcd
        from scipy.signal import resample_poly
        g = gcd(int(sr), int(target_sr))
        return resample_poly(a.astype(np.float32), int(target_sr) // g, int(sr) // g).astype(np.float32)

    @classmethod
    def _load_audio_to_np(cls, x: str) -> Tuple[np.ndarray, int]:
        """wav path, URL or base64 (raw / data URL) -> (mono float32 waveform, its sampling rate).  PCM / float WAV only
        (scipy.io.wavfile; the reference's soundfile / librosa also read flac, ogg, mp3)."""
        import base64
        import io
        from scipy.io import wavfile
        if cls._is_url(x):
            import urllib.request
            with urllib.request.urlopen(x) as resp:
                src = io.BytesIO(resp.read())
        elif cls._is_probably_base64(x):
            if "," in x and x.strip().startswith("data:"):
                x = x.split(",", 1)[1]
            src = io.BytesIO(base64.b64decode(x))
        else:
            src = x
        sr, audio = wavfile.read(src)
        if audio.dtype.kind == "i":
            audio = audio.astype(np.float32) / float(np.iinfo(audio.dtype).max + 1)
        elif audio.dtype.kind == "u":  # 8-bit PCM is unsigned
            audio = (audio.astype(np.float32) - 128.0) / 128.0
        audio = audio.astype(np.float32)
        if audio.ndim > 1:
            audio = np.mean(audio, axis=-1).astype(np.float32)
        return audio, int(sr)

    @classmethod
    def load_audio(cls, x: str, target_sr: int) -> np.ndarray:
        """:121-157 — wav path, URL or base64 -> mono float32 at target_sr."""
        audio, sr = cls._load_audio_to_np(x)
        return cls._resample(audio, sr, target_sr)

    @classmethod
    def _normalize_audio_inputs(cls, audios, sr, target_sr=24000) -> List[np.ndarray]:
        """:159-207 — str | ndarray | list of either -> list of 1-D float32 waveforms at target_sr."""
        if isinstance(audios, (str, np.ndarray)):
            audios = [audios]
        if len(audios) == 0:
            return []
        if isinstance(audios[0], str):
            return [cls.load_audio(x, target_sr) for x in audios]
        if sr is None:
            raise ValueError("For numpy waveform input, you must provide `sr` (original sampling rate).")
        out = []
        for a in audios:
            if not isinstance(a, np.ndarray):
                raise TypeError("Mixed input types are not supported. Use all paths/base64 or all numpy arrays.")
            if a.ndim > 1:
                a = np.mean(a, axis=-1)
            out.append(cls._resample(a.astype(np.float32), int(sr), target_sr))
        return out

    def encode(self, audios, sr=None, return_dict=True):
        """:208-257 -> Qwen3TTSTokenizerV2Model.encode (…v2.py:961-991): returns an object with
        `.audio_codes = List[LongTensor (T_i, 16)]` on the device (or the 1-tuple when return_dict=False)."""
        if self.encoder is None:
            raise RuntimeError("this tokenizer was built without encoder weights (decode-only)")
        wavs = self._normalize_audio_inputs(audios, sr, self.get_input_sample_rate())
        codes = self.encoder.encode([torch.from_numpy(w) for w in wavs])
        if not return_dict:
            return (codes,)
        from types import SimpleNamespace
        return SimpleNamespace(audio_codes=codes)

    def open_encode_stream(self, batch: int = 1, max_packet_frames: int = 8, sample_rate=None):
        """A streaming encoder of `batch` rows (codec_encoder.EncoderStream): push({row: samples}) returns the (n_i, 16)
        codes of the frames each push completes, end(rows) the clip's last frame, in the layout of encode().audio_codes;
        a clip's pushes plus its end equal encode() of the whole clip.  `sample_rate`: the rate of the pushed audio
        (None: get_input_sample_rate()).  At another supported rate (audio.SUPPORTED_RATES) the pushes are resampled on
        the GPU as they arrive (audio.ResampledEncoderStream), and a clip's codes equal
        encoder.forward(Resampler.oneshot(clip)) bit for bit.  encode(..., sr=) keeps resampling on the host with
        scipy.signal.resample_poly: the same filter and sum in another rounding order, so its waveform agrees with the
        GPU's to within 1e-5, and the codes of the two may differ only where the RVQ has a near-tie."""
        if self.encoder is None:
            raise RuntimeError("this tokenizer was built without encoder weights (decode-only)")
        return self.encoder.open_stream(batch, max_packet_frames, sample_rate=sample_rate)

    def decode(self, encoded) -> Tuple[List[np.ndarray], int]:
        """:259-365 — accepts an encode()-style output (has .audio_codes), a dict or a list of dicts whose
        "audio_codes" is a (T,K) tensor / ndarray; pads with -1, decodes, trims to T_i*1920, returns float32 numpy."""
        if hasattr(encoded, "audio_codes"):
            codes_in = encoded.audio_codes
        elif isinstance(encoded, dict):
            if "audio_codes" not in encoded:
                raise ValueError("`encoded` dict must contain 'audio_codes'.")
            codes_in = encoded["audio_codes"]
        elif isinstance(encoded, list):
            codes_in = [e["audio_codes"] for e in encoded]
        else:
            raise TypeError("`encoded` must be an encode output, a dict, or a list of dicts.")
        if isinstance(codes_in, torch.Tensor):
            # :312-322 — a single (T, K) sample is unsqueezed, a 3-D tensor is an already padded (B, T, K) batch
            t = codes_in
            if t.dim() == 2:
                t = t.unsqueeze(0)
            if t.dim() != 3:
                raise ValueError(f"audio_codes tensor must have shape (T, K) or (B, T, K), got {tuple(t.shape)}")
            ac = t.to(self.device, torch.long)
        else:
            tens = []
            for c in codes_in:  # :323-326 — list of per-sample tensors / arrays, right-padded with -1
                c = c if isinstance(c, torch.Tensor) else torch.from_numpy(np.asarray(c))
                if c.dim() != 2:
                    raise ValueError(f"audio_codes must have shape (T, K), got {tuple(c.shape)}")
                tens.append(c.to(self.device, torch.long))
            if not tens:
                return [], int(self.get_output_sample_rate())
            Tm = max(int(c.shape[0]) for c in tens)
            ac = torch.full((len(tens), max(Tm, 1), tens[0].shape[1]), -1, dtype=torch.long, device=self.device)
            for i, c in enumerate(tens):
                ac[i, :c.shape[0]] = c
        wavs = []
        mb = max(int(getattr(self.decoder, "max_batch", ac.shape[0])), 1)
        for s0 in range(0, ac.shape[0], mb):  # tile by the codec engine's batch capacity (like model.generate)
            wavs += self.decoder.decode(ac[s0:s0 + mb])
        return [w.to(torch.float32).detach().cpu().numpy() for w in wavs], int(self.get_output_sample_rate())


class Qwen3TTSModel:
    """inference/qwen3_tts_model.py:54 — same entry points, input normalisation, kwarg precedence and returns."""

    def __init__(self, model: Qwen3TTSForConditionalGenerationB200, processor, generate_defaults: Optional[dict] = None):
        self.model = model
        self.processor = processor
        self.generate_defaults = generate_defaults or {}
        self.device = model.device

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, device_map="cuda:0", processor=None, max_batch=32,
                        max_ctx=4096, codec_max_frames=1024, **kwargs) -> "Qwen3TTSModel":
        """inference/qwen3_tts_model.py:82-121 + core/models/modeling_qwen3_tts.py:1843-1941: model weights, the
        `speech_tokenizer/` sub-directory, `generation_config.json` (-> generate_defaults) and the text processor
        (AutoTokenizer of the same directory, called like Qwen3TTSProcessor.__call__, processing_qwen3_tts.py:46-75).
        `dtype` / `attn_implementation` are accepted and ignored; `processor=` overrides the tokenizer (tests)."""
        from . import checkpoint
        d = checkpoint.resolve_dir(pretrained_model_name_or_path)
        device = device_map if isinstance(device_map, (str, torch.device)) else "cuda:0"
        tcfg, W, meta, gen = checkpoint.load_tts_checkpoint(d, device=device)
        core = Qwen3TTSForConditionalGenerationB200(
            tcfg, W, device=device, spk_id=meta["spk_id"], spk_is_dialect=meta["spk_is_dialect"],
            codec_language_id=meta["codec_language_id"], tts_model_type=meta["tts_model_type"] or "custom_voice",
            tts_model_size=meta["tts_model_size"] or "1b7", max_batch=max_batch, max_ctx=max_ctx)
        st_dir = os.path.join(d, "speech_tokenizer")
        if not os.path.isdir(st_dir):
            raise ValueError(f"{d}/speech_tokenizer not exists")
        core.load_speech_tokenizer(Qwen3TTSTokenizer.from_pretrained(st_dir, device_map=device, max_frames=codec_max_frames))
        core.load_generate_config(gen or {})
        core.tokenizer_type = meta.get("tokenizer_type")
        if meta.get("speaker_encoder_weights"):
            from .speaker_encoder import SpeakerEncoder
            core.load_speaker_encoder(SpeakerEncoder(meta["speaker_encoder_config"], meta["speaker_encoder_weights"], device=device))
        if processor is None:
            from transformers import AutoTokenizer
            tok = AutoTokenizer.from_pretrained(d)

            def processor(text=None, **kw):
                if text is None:
                    raise ValueError("You need to specify either a `text` input to process.")
                return tok(text if isinstance(text, list) else [text], **kw)
        return cls(model=core, processor=processor, generate_defaults=core.generate_config)

    # ---- helpers (:207-352)
    @staticmethod
    def _ensure_list(x):
        return x if isinstance(x, list) else [x]

    @staticmethod
    def _build_assistant_text(text):
        return f"<|im_start|>assistant\n{text}<|im_end|>\n<|im_start|>assistant\n"

    @staticmethod
    def _build_ref_text(text):
        return f"<|im_start|>assistant\n{text}<|im_end|>\n"

    @staticmethod
    def _build_instruct_text(instruct):
        return f"<|im_start|>user\n{instruct}<|im_end|>\n"

    def _tokenize_texts(self, texts):
        out = []
        for text in texts:
            ids = self.processor(text=text, return_tensors="pt", padding=True)["input_ids"].to(self.device)
            out.append(ids.unsqueeze(0) if ids.dim() == 1 else ids)
        return out

    def _merge_generate_kwargs(self, **kw) -> Dict[str, Any]:
        hard = dict(do_sample=True, top_k=50, top_p=1.0, temperature=0.9, repetition_penalty=1.05,
                    subtalker_dosample=True, subtalker_top_k=50, subtalker_top_p=1.0, subtalker_temperature=0.9,
                    max_new_tokens=2048)
        merged = {k: v for k, v in kw.items() if k not in hard}
        for name, dv in hard.items():
            uv = kw.get(name)
            merged[name] = uv if uv is not None else self.generate_defaults.get(name, dv)
        return merged

    def _supported_languages_set(self):
        s = self.model.get_supported_languages()
        return None if s is None else {x.lower() for x in s}

    def _supported_speakers_set(self):
        s = self.model.get_supported_speakers()
        return None if s is None else {x.lower() for x in s}

    def _validate_languages(self, languages):
        sup = self._supported_languages_set()
        if sup is None:
            return
        bad = [l for l in languages if l is None or l.lower() not in sup]
        if bad:
            raise ValueError(f"Unsupported languages: {bad}. Supported: {sorted(sup)}")

    def _validate_speakers(self, speakers):
        sup = self._supported_speakers_set()
        if sup is None:
            return
        bad = [s for s in speakers if s is not None and s != "" and s.lower() not in sup]
        if bad:
            raise ValueError(f"Unsupported speakers: {bad}. Supported: {sorted(sup)}")

    def get_supported_speakers(self):
        s = self._supported_speakers_set()
        return None if s is None else sorted(s)

    def get_supported_languages(self):
        s = self._supported_languages_set()
        return None if s is None else sorted(s)

    def _broadcast(self, texts, *lists):
        out = []
        for l in lists:
            if len(l) == 1 and len(texts) > 1:
                l = l * len(texts)
            out.append(l)
        return out

    def _decode(self, codes_list):
        return self.model.speech_tokenizer.decode([{"audio_codes": c} for c in codes_list])

    # ---- :731-839
    def generate_custom_voice(self, text, speaker, language=None, instruct=None, non_streaming_mode=True, **kwargs):
        if self.model.tts_model_type != "custom_voice":
            raise ValueError(f"model type {self.model.tts_model_type} does not support generate_custom_voice")
        texts = self._ensure_list(text)
        languages = self._ensure_list(language) if isinstance(language, list) else (
            [language] * len(texts) if language is not None else ["Auto"] * len(texts))
        speakers = self._ensure_list(speaker)
        if self.model.tts_model_size in "0b6":
            instruct = None
        instructs = self._ensure_list(instruct) if isinstance(instruct, list) else (
            [instruct] * len(texts) if instruct is not None else [""] * len(texts))
        languages, speakers, instructs = self._broadcast(texts, languages, speakers, instructs)
        if not (len(texts) == len(languages) == len(speakers) == len(instructs)):
            raise ValueError(f"Batch size mismatch: text={len(texts)}, language={len(languages)}, "
                             f"speaker={len(speakers)}, instruct={len(instructs)}")
        self._validate_languages(languages)
        self._validate_speakers(speakers)
        input_ids = self._tokenize_texts([self._build_assistant_text(t) for t in texts])
        instruct_ids = [None if (i is None or i == "") else self._tokenize_texts([self._build_instruct_text(i)])[0]
                        for i in instructs]
        codes, _ = self.model.generate(input_ids=input_ids, instruct_ids=instruct_ids, languages=languages,
                                       speakers=speakers, non_streaming_mode=non_streaming_mode,
                                       **self._merge_generate_kwargs(**kwargs))
        return self._decode(codes)

    # ---- live text (speaking a text while it is still being written)
    def build_live_request(self, text, speaker=None, language=None, instruct=None, voice_clone_prompt=None):
        """One live request for ContinuousBatcher.submit(..., text_open=True): (inputs_embeds, trailing_text,
        tts_pad_embed) of the streaming layout for the text known so far (`text`, at least one token).  Custom voice
        (`speaker`, optional `instruct`), voice design (`instruct`) and x-vector-only voice-clone prompts are supported;
        an ICL prompt raises ValueError.  Feed later pieces with append_text(rid, live_text_rows(piece)) and end with
        append_text(rid, live_text_end()) and close_text(rid).  The request then generates what the whole text's ids
        generate up front (non_streaming_mode=False).  The guarantee is in ids: a string split into pieces may tokenise
        differently from the whole string."""
        if isinstance(text, list):
            raise ValueError("build_live_request takes one text")
        if voice_clone_prompt is not None:
            input_ids, _, vcp, languages = self._voice_clone_inputs(text, language, None, None, False, voice_clone_prompt,
                                                                    "build_live_request")
            embeds, trailing, pad = self.model.build_live_prefill(input_ids, voice_clone_prompt=vcp, languages=languages)
            return embeds[0], trailing[0], pad
        language = "Auto" if language is None else language
        self._validate_languages([language])
        self._validate_speakers([speaker])
        if self.model.tts_model_type == "custom_voice" and self.model.tts_model_size in "0b6":
            instruct = None
        input_ids = self._tokenize_texts([self._build_assistant_text(text)])
        instruct_ids = [None if (instruct is None or instruct == "") else self._tokenize_texts([self._build_instruct_text(instruct)])[0]]
        embeds, trailing, pad = self.model.build_live_prefill(input_ids, instruct_ids=instruct_ids, languages=[language],
                                                              speakers=[speaker])
        return embeds[0], trailing[0], pad

    def build_live_clone_request(self, text, voice_clone_prompt=None, voice: Optional["Voice"] = None, language=None):
        """One live request of an ICL voice clone for ContinuousBatcher.submit(inputs_embeds, trailing_text,
        text_open=True, overlay=overlay, ref_codes= / voice=): (inputs_embeds, trailing_text, tts_pad_embed, overlay) of
        the streaming layout for the text known so far (`text`, which may be empty).  Either `voice_clone_prompt`, one
        ICL item (with ref_codes=item.ref_code at submit), or `voice`, an ICL voice registered with
        non_streaming_mode=False, whose inputs_embeds are the rows after voice.prefix as build_voice_request returns
        them (the voice fixes the language).  The prompt's last K = max(0, Lc - R) positions overlay the reference's
        last frames with target text (Lc = 1 + reference frames, R = reference text tokens), so the request is admitted
        once K text rows have arrived or its text is closed (Qwen3TTSForConditionalGenerationB200.build_live_icl_prefill).
        Feed it as any live request (live_text_rows, live_text_end, close_text); it then generates what the whole
        text's ids generate up front (non_streaming_mode=False).  Other prompts and voices take build_live_request and
        build_voice_request(live=True)."""
        if isinstance(text, list):
            raise ValueError("build_live_clone_request takes one text")
        if (voice is None) == (voice_clone_prompt is None):
            raise ValueError("build_live_clone_request takes one of voice_clone_prompt and voice")
        if voice is not None:
            if voice.closed:
                raise ValueError("the voice is closed")
            if not voice.icl:
                raise ValueError("not an ICL voice: a live request of it takes build_voice_request(text, voice, live=True)")
            if voice.non_streaming_mode:
                raise ValueError("live text needs a voice registered with non_streaming_mode=False (the non-streaming ICL "
                                 "layout puts the whole text before the reference codes)")
            if language is not None:
                raise ValueError("a registered voice fixes its language")
            input_ids = self._tokenize_texts([self._build_assistant_text(text)])
            e, t, p, o = self.model.build_live_icl_prefill(input_ids, voice.ref_ids, voice.vcp, [voice.language])
            return e[0][voice.prefix_len:], t[0], p, o[0]
        items = voice_clone_prompt if isinstance(voice_clone_prompt, list) else [voice_clone_prompt]
        if len(items) != 1 or not isinstance(items[0], VoiceClonePromptItem):
            raise ValueError("build_live_clone_request takes one VoiceClonePromptItem")
        if items[0].ref_code is None or not items[0].icl_mode:
            raise ValueError("not an ICL voice-clone prompt: a live request of it takes build_live_request")
        input_ids, ref_ids, vcp, languages = self._voice_clone_inputs(text, language, None, None, False, items,
                                                                      "build_live_clone_request")
        e, t, p, o = self.model.build_live_icl_prefill(input_ids, ref_ids, vcp, languages)
        return e[0], t[0], p, o[0]

    def live_text_rows(self, text: str) -> torch.Tensor:
        """Trailing rows (n, H) of one more piece of a live request's text: its token ids with no chat wrapper."""
        ids = self.processor(text=text, return_tensors="pt", padding=True)["input_ids"]
        return self.model.text_rows(ids.reshape(-1))

    def live_text_end(self) -> torch.Tensor:
        """The (1, H) tts_eos row to append_text before close_text: it tells the model the text is over."""
        return self.model.tts_eos_row()

    # ---- :636-728
    def generate_voice_design(self, text, instruct, language=None, non_streaming_mode=True, **kwargs):
        if self.model.tts_model_type != "voice_design":
            raise ValueError(f"model type {self.model.tts_model_type} does not support generate_voice_design")
        texts = self._ensure_list(text)
        languages = self._ensure_list(language) if isinstance(language, list) else (
            [language] * len(texts) if language is not None else ["Auto"] * len(texts))
        instructs = self._ensure_list(instruct)
        languages, instructs = self._broadcast(texts, languages, instructs)
        if not (len(texts) == len(languages) == len(instructs)):
            raise ValueError(f"Batch size mismatch: text={len(texts)}, language={len(languages)}, instruct={len(instructs)}")
        self._validate_languages(languages)
        input_ids = self._tokenize_texts([self._build_assistant_text(t) for t in texts])
        instruct_ids = [None if (i is None or i == "") else self._tokenize_texts([self._build_instruct_text(i)])[0]
                        for i in instructs]
        codes, _ = self.model.generate(input_ids=input_ids, instruct_ids=instruct_ids, languages=languages,
                                       non_streaming_mode=non_streaming_mode, **self._merge_generate_kwargs(**kwargs))
        return self._decode(codes)

    # ---- :207-257 — str (path / URL / base64) | (ndarray, sr) | list of those -> [(float32 mono waveform, sr)]
    def _normalize_audio_inputs(self, audios) -> List[Tuple[np.ndarray, int]]:
        items = audios if isinstance(audios, list) else [audios]
        out: List[Tuple[np.ndarray, int]] = []
        for a in items:
            if isinstance(a, str):
                out.append(Qwen3TTSTokenizer._load_audio_to_np(a))
            elif isinstance(a, tuple) and len(a) == 2 and isinstance(a[0], np.ndarray):
                out.append((a[0].astype(np.float32), int(a[1])))
            elif isinstance(a, np.ndarray):
                raise ValueError("For numpy waveform input, pass a tuple (audio, sr).")
            else:
                raise TypeError(f"Unsupported audio input type: {type(a)}")
        return [(np.mean(w, axis=-1).astype(np.float32) if w.ndim > 1 else w, sr) for w, sr in out]

    # ---- :355-458
    def create_voice_clone_prompt(self, ref_audio, ref_text=None, x_vector_only_mode=False) -> List[VoiceClonePromptItem]:
        if self.model.tts_model_type != "base":
            raise ValueError(f"model with \ntokenizer_type: {getattr(self.model, 'tokenizer_type', None)}\n"
                             f"tts_model_size: {self.model.tts_model_size}\ntts_model_type: {self.model.tts_model_type}\n"
                             "does not support create_voice_clone_prompt, Please check Model Card or Readme for more details.")
        audios = self._ensure_list(ref_audio)
        texts = self._ensure_list(ref_text) if isinstance(ref_text, list) else [ref_text] * len(audios)
        xvecs = self._ensure_list(x_vector_only_mode) if isinstance(x_vector_only_mode, list) else [x_vector_only_mode] * len(audios)
        if len(texts) != len(audios) or len(xvecs) != len(audios):
            raise ValueError(f"Batch size mismatch: ref_audio={len(audios)}, ref_text={len(texts)}, x_vector_only_mode={len(xvecs)}")
        normalized = self._normalize_audio_inputs(audios)
        srs = [sr for _, sr in normalized]
        tok = self.model.speech_tokenizer
        if len(set(srs)) == 1:
            ref_codes = tok.encode([w for w, _ in normalized], sr=srs[0]).audio_codes
        else:
            ref_codes = [tok.encode(w, sr=sr).audio_codes[0] for w, sr in normalized]
        items: List[VoiceClonePromptItem] = []
        for i, ((wav, sr), code, rtext, xv) in enumerate(zip(normalized, ref_codes, texts, xvecs)):
            if not xv and (rtext is None or rtext == ""):
                raise ValueError(f"ref_text is required when x_vector_only_mode=False (ICL mode). Bad index={i}")
            target = int(self.model.speaker_encoder_sample_rate)
            w24 = wav if sr == target else Qwen3TTSTokenizer._resample(wav, sr, target)
            emb = self.model.extract_speaker_embedding(audio=w24, sr=target)
            items.append(VoiceClonePromptItem(ref_code=None if xv else code, ref_spk_embedding=emb,
                                              x_vector_only_mode=bool(xv), icl_mode=bool(not xv), ref_text=rtext))
        return items

    @staticmethod
    def _prompt_items_to_voice_clone_prompt(items: List[VoiceClonePromptItem]) -> Dict[str, Any]:
        return dict(ref_code=[it.ref_code for it in items], ref_spk_embedding=[it.ref_spk_embedding for it in items],
                    x_vector_only_mode=[it.x_vector_only_mode for it in items], icl_mode=[it.icl_mode for it in items])

    # ---- :469-633
    def _voice_clone_inputs(self, text, language, ref_audio, ref_text, x_vector_only_mode, voice_clone_prompt, caller):
        """generate_voice_clone's input handling (:469-603): list-ify and broadcast, validate, build the prompt from
        raw audio when none is given, tokenise.  Returns (input_ids, ref_ids, voice_clone_prompt dict, languages)."""
        if self.model.tts_model_type != "base":
            raise ValueError(f"model type {self.model.tts_model_type} does not support {caller}")
        texts = self._ensure_list(text)
        languages = self._ensure_list(language) if isinstance(language, list) else (
            [language] * len(texts) if language is not None else ["Auto"] * len(texts))
        (languages,) = self._broadcast(texts, languages)
        if len(texts) != len(languages):
            raise ValueError(f"Batch size mismatch: text={len(texts)}, language={len(languages)}")
        self._validate_languages(languages)
        if voice_clone_prompt is None:
            if ref_audio is None:
                raise ValueError("Either `voice_clone_prompt` or `ref_audio` must be provided.")
            voice_clone_prompt = self.create_voice_clone_prompt(ref_audio, ref_text, x_vector_only_mode)
        if isinstance(voice_clone_prompt, list):
            items = voice_clone_prompt
            if len(items) == 1 and len(texts) > 1:
                items = items * len(texts)
            if len(items) != len(texts):
                raise ValueError(f"Batch size mismatch: prompt={len(items)}, text={len(texts)}")
            vcp = self._prompt_items_to_voice_clone_prompt(items)
            ref_texts = [it.ref_text for it in items]
        else:
            vcp, ref_texts = voice_clone_prompt, None
        input_ids = self._tokenize_texts([self._build_assistant_text(t) for t in texts])
        ref_ids = None
        if ref_texts is not None:
            ref_ids = [None if (rt is None or rt == "") else self._tokenize_texts([self._build_ref_text(rt)])[0]
                       for rt in ref_texts]
        return input_ids, ref_ids, vcp, languages

    # ---- registered voices: a voice's prompt prefix and reference state are computed once and kept on the device
    def register_voice(self, speaker=None, language=None, instruct=None, voice_clone_prompt=None,
                       non_streaming_mode=False) -> "Voice":
        """Register a voice for ContinuousBatcher.submit(..., voice=): the rows of its prompt that do not depend on a
        request's text (the instruct, the role rows, the codec-prefix overlay and, for an ICL clone, the reference
        positions before the target text) are prefilled once into a prefix of the AR engine, and an ICL clone's
        reference codes are decoded once into a row of the codec's reference bank.  The arguments and their checks are
        those of generate_custom_voice (speaker, instruct), generate_voice_design (instruct) and generate_voice_clone
        (one voice_clone_prompt item), by model type.  An ICL prefix depends on the layout, so the voice fixes
        `non_streaming_mode`.  Build its requests with build_voice_request; Voice.close() releases it."""
        mt = self.model.tts_model_type
        language = "Auto" if language is None else language
        if isinstance(language, list) or isinstance(speaker, list) or isinstance(instruct, list):
            raise ValueError("register_voice takes one voice")
        vcp, ref_ids, icl = None, None, False
        if mt == "base":
            if voice_clone_prompt is None:
                raise ValueError("a base model's voice needs a voice_clone_prompt")
            items = voice_clone_prompt if isinstance(voice_clone_prompt, list) else [voice_clone_prompt]
            if len(items) != 1:
                raise ValueError(f"register_voice takes one voice_clone_prompt item, got {len(items)}")
            self._validate_languages([language])
            vcp = self._prompt_items_to_voice_clone_prompt(items)
            icl = items[0].ref_code is not None and bool(items[0].icl_mode)
            if icl:
                ref_ids = [self._tokenize_texts([self._build_ref_text(items[0].ref_text)])[0]]
            speaker, instruct = None, None
        elif mt == "custom_voice":
            self._validate_languages([language])
            self._validate_speakers([speaker])
            if self.model.tts_model_size in "0b6":
                instruct = None
        elif mt == "voice_design":
            self._validate_languages([language])
            speaker = None
        else:
            raise ValueError(f"model type {mt} does not support register_voice")
        if voice_clone_prompt is not None and mt != "base":
            raise ValueError(f"model type {mt} takes no voice_clone_prompt")
        instruct_ids = [None if (instruct is None or instruct == "") else self._tokenize_texts([self._build_instruct_text(instruct)])[0]]
        voice = Voice(self, language, speaker, instruct_ids, vcp, ref_ids, bool(non_streaming_mode), icl)
        # the prompt of any text: its first rows are the voice's, computed here once
        embeds, _, _, T = self._voice_rows(voice, "a")
        voice.prefix = embeds[:self._voice_prefix_len(voice, embeds.shape[0], T)].clone()
        eng = self.model.engine
        voice.prefix_id = eng.create_prefix(voice.prefix)
        if icl:
            tok = self.model.speech_tokenizer
            dec = getattr(tok, "decoder", None) if tok is not None else None
            if dec is None:
                eng.free_prefix(voice.prefix_id)
                raise ValueError("an ICL voice needs the model's speech tokenizer to keep its reference state")
            voice.codec, voice.ref_codes = dec, vcp["ref_code"][0]
            voice.bank = dec.bank_reference(voice.ref_codes)
        return voice

    def _voice_rows(self, voice: "Voice", text, live=False):
        """build_prefill (or build_live_prefill) of one request of `voice` speaking `text`, and the text's tokens."""
        input_ids = self._tokenize_texts([self._build_assistant_text(text)])
        T = int(input_ids[0].reshape(-1).shape[0]) - 8                 # 3 role and 5 closing tokens around the text
        if live:
            e, t, p = self.model.build_live_prefill(input_ids, instruct_ids=voice.instruct_ids, voice_clone_prompt=voice.vcp,
                                                    languages=[voice.language], speakers=[voice.speaker])
        else:
            e, t, p = self.model.build_prefill(input_ids, voice.instruct_ids, voice.ref_ids, voice.vcp, [voice.language],
                                               [voice.speaker], voice.non_streaming_mode)
        return e[0], t[0], p, T

    def _voice_prefix_len(self, voice: "Voice", n_rows: int, T: int) -> int:
        """Rows of the prompt layout (_plan_sample) that do not depend on the text, never the prompt's last row: the
        instruct, 3 role and |C|-1 overlay rows, and for an ICL clone the first min(R, Lc) (streaming) or R
        (non-streaming) ICL positions, R the reference text's tokens and Lc = L + 1 the codec stream.  `n_rows`: the
        prompt length of a request whose text has T tokens."""
        if not voice.icl:
            return n_rows - (T + 2 if voice.non_streaming_mode else 1)    # the text rows: T + 2, or the first token
        R = int(voice.ref_ids[0].reshape(-1).shape[0]) - 5              # ref_id[3:-2]
        Lc = int(voice.vcp["ref_code"][0].shape[0]) + 1
        if voice.non_streaming_mode:
            return n_rows - (R + T + 1) - Lc + R                          # text stream R + T + 1 rows, then Lc
        return min(n_rows - Lc + min(R, Lc), n_rows - 1)

    def build_voice_request(self, text, voice: "Voice", live: bool = False):
        """One request of a registered voice for ContinuousBatcher.submit(suffix_embeds, trailing, voice=voice):
        (suffix_embeds, trailing_text, tts_pad_embed), where cat(voice.prefix, suffix_embeds) and trailing_text are
        the rows build_prefill makes for the same request.  With `live=True` the trailing rows end without tts_eos,
        as in build_live_request (submit with text_open=True); ICL voices refuse it (build_live_clone_request)."""
        if voice.closed:
            raise ValueError("the voice is closed")
        if isinstance(text, list):
            raise ValueError("build_voice_request takes one text")
        if live and voice.non_streaming_mode:
            raise ValueError("live text needs a voice registered with non_streaming_mode=False")
        if live and voice.icl:
            raise ValueError("a live request of an ICL voice takes build_live_clone_request")
        embeds, trailing, pad, _ = self._voice_rows(voice, text, live)
        return embeds[voice.prefix_len:], trailing, pad

    def build_voice_clone_requests(self, text, language=None, ref_audio=None, ref_text=None, x_vector_only_mode=False,
                                   voice_clone_prompt=None, non_streaming_mode=False):
        """generate_voice_clone's inputs as requests for the streaming paths (ContinuousBatcher.submit,
        TTSEngine.stream_synthesize): ([(inputs_embeds, trailing_text, ref_code or None)] per text, tts_pad_embed).
        A request's ref_code is what generate_voice_clone decodes in front of its codes; pass it as `ref_codes` so the
        streamed audio is the part generate_voice_clone keeps."""
        input_ids, ref_ids, vcp, languages = self._voice_clone_inputs(text, language, ref_audio, ref_text, x_vector_only_mode,
                                                                      voice_clone_prompt, "build_voice_clone_requests")
        embeds, trailing, pad = self.model.build_prefill(input_ids, ref_ids=ref_ids, voice_clone_prompt=vcp, languages=languages,
                                                         non_streaming_mode=non_streaming_mode)
        ref_codes = vcp.get("ref_code", None)
        refs = [None if ref_codes is None else ref_codes[i] for i in range(len(embeds))]
        return list(zip(embeds, trailing, refs)), pad

    def generate_voice_clone(self, text, language=None, ref_audio=None, ref_text=None, x_vector_only_mode=False,
                             voice_clone_prompt=None, non_streaming_mode=False, **kwargs):
        input_ids, ref_ids, vcp, languages = self._voice_clone_inputs(text, language, ref_audio, ref_text, x_vector_only_mode,
                                                                      voice_clone_prompt, "generate_voice_clone")
        codes, _ = self.model.generate(input_ids=input_ids, ref_ids=ref_ids, voice_clone_prompt=vcp, languages=languages,
                                       non_streaming_mode=non_streaming_mode, **self._merge_generate_kwargs(**kwargs))
        ref_codes = vcp.get("ref_code", None)
        full = []
        for i, c in enumerate(codes):
            if ref_codes is not None and ref_codes[i] is not None:
                full.append(torch.cat([ref_codes[i].to(c.device), c], dim=0))
            else:
                full.append(c)
        wavs, fs = self._decode(full)
        out = []
        for i, wav in enumerate(wavs):
            if ref_codes is not None and ref_codes[i] is not None:
                cut = int(int(ref_codes[i].shape[0]) / max(int(full[i].shape[0]), 1) * wav.shape[0])
                out.append(wav[cut:])
            else:
                out.append(wav)
        return out, fs
