"""Calibration of the full-shape parity tolerance: PyTorch bf16 (the reference's own arithmetic) vs fp32, teacher-forced,
1.7B shapes, ctx 200-230, 8 frames.  The GPU engine is held to 1.5x the max gap printed here (tests/test_gpu_ar.py)."""
import os, sys, time, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import talker as OT
from tests import helpers as Hh
torch.set_num_threads(8)
cfg = OT.cfg_1p7b(); cfg.text_vocab_size = 1000
W = OT.random_weights(cfg, seed=28, with_text=False)
Wb, Wf = Hh.bf16_weights(W); del W
lens = [230, 203]
embs, trail, pad = Hh.make_inputs(cfg, lens, [0, 3], seed=29)
N = 8
sp = OT.SamplingCfg(do_sample=False, subtalker_dosample=False, max_new_tokens=N + 1, suppress_eos=True)
t0 = time.time()
ref = OT.generate(Wf, cfg, [e.float() for e in embs], [t.float() for t in trail], pad.float(), sp, record_logits=True)
print("fp32 oracle", time.time() - t0, flush=True)
forced = torch.stack(ref.codes).numpy()
t0 = time.time()
rb = OT.generate(Wb, cfg, embs, trail, pad, sp, record_logits=True, forced_codes=forced)
print("bf16 oracle", time.time() - t0, flush=True)
G = cfg.num_code_groups
for f in range(N + 1):
    a, b = ref.record["talker_logits"][f], np.asarray(rb.record["talker_logits"][f], dtype=np.float32)
    s = a.std(); d = np.abs(a - b)
    print("talker frame", f, "max/std %.3f mean/std %.4f" % (d.max() / s, d.mean() / s), flush=True)
worst = wmean = 0
for f in range(N):
    for j in range(G - 1):
        a, b = ref.record["cp_logits"][f * (G - 1) + j], np.asarray(rb.record["cp_logits"][f * (G - 1) + j], dtype=np.float32)
        worst = max(worst, np.abs(a - b).max() / a.std()); wmean = max(wmean, np.abs(a - b).mean() / a.std())
print("cp worst max/std %.3f  worst mean/std %.4f" % (worst, wmean))
