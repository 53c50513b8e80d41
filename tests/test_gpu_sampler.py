"""Direct checks of the frame-step kernel's sample phase (csrc/ar_sampler.cuh) against oracle/sampler.py, row by row, at its
fast-path, radix-select, top-p, tie, CDF and bookkeeping edges.

The phase is run through tests/csrc/sampler_shim.cu: a test-only kernel that calls sample_phase() one CTA per row, as
q3_step_kernel does.  The shim compiles its own copy of the phase from the shipped source under the library's flags (the
__noinline__ helpers sample_fast, kth_largest, block_reduce and block_min_int are the same source); the instantiation
inside q3_step_kernel is checked by tests/test_gpu_ar.py::test_sampler_against_oracle_on_engine_logits.

Acceptance rule.  No fast-math flag is set, so the processed scores (penalty, temperature: correctly rounded fp32 * and /)
are bit-identical to the oracle's.  Hence:
- greedy rows: the token equals the oracle's (first maximum, like torch.argmax);
- every sampled token lies in the oracle's kept set (top-k exact, ties included);
- inverse CDF: the token equals the one of the fp64 CDF C_j = sum_{i<=j} p_i, p_i = exp(d_i), d_i = fl32(s_i - max) (the
  kernel's own fp32 difference), target u * C_last, unless every CDF boundary between the two tokens lies within
      bound = (1 + u) * E + 2^-24 * u * T,   E = sum_i eps_i * p_i + (m - 1) * 2^-24 * T + m * 2^-126,
      eps_i = (3 + floor(1.173 |d_i|)) * 2^-23
  of u * T (T = C_last, m = kept tokens).  eps_i is __expf's documented error of 2 + floor(1.173 |x|) ulp plus one ulp for
  the oracle's own float32 exp, (m - 1) 2^-24 T bounds an fp32 sum of m non-negative terms in any order, m 2^-126 the
  flush to zero of subnormal results, and the last term the rounding of the target u * total.  The oracle's token
  (sample_from_scores) is held to the same rule.
- top-p: a token is removed iff its fp64 ascending cumulative share (ties in id order) is <= 1 - p, unless that share
  lies within 2 E / T + 2^-23 of the kernel's fp32 threshold 1.0f - p or the oracle's fp32(1 - p) (or between them);
  such tokens may go either way, and the draw must then match the inverse CDF of one of the resulting kept sets.
- "grid" rows keep only equal scores, so every kept p is __expf(0) = 1 exactly, the partial sums are small integers
  and u is a multiple of 1/64 (row keys found by a numpy port of oracle/philox.py): there E = 0 and the target is exact,
  so boundary draws (run > target, never >=) and top-p at exactly 1 - p are checked bit for bit.
Bookkeeping (finished, n_valid, n_gen, c0, cur, seen, codes_out, the next inputs of the code predictor and the talker)
is compared bit-exactly, and every buffer the phase indexes by token has guard rows that must stay untouched.
"""
import ctypes as C
import functools
import math
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

from oracle import philox
from oracle import sampler as OS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "csrc", "sampler_shim.cu")

V_T, EOS, V_C = 3072, 2150, 2048   # talker vocabulary with its EOS and suppress range [V-1024, V); code predictor
H, G, WN, TS, CS = 64, 16, 32, 4, 6  # hidden, code groups, cp next-row width, trailing stride, codes_out stride
SEEN_GUARD, SENT_BF16, SENT_CODE = 0x5A, 0x7FAB, -9
KEYS = 1 << 22
STATS = {"sampled": 0, "near_boundary": 0, "topp_ambiguous": 0, "grid_draws": 0}
NEG = -np.inf


# ================================================================================================ Philox (numpy port)
def philox_u24(seed, keys, frame, group):
    """(philox4x32_10(seed; key, frame, group, 0)[0] >> 8) for an array of row keys: u = result / 2^24."""
    M = np.uint64(0xFFFFFFFF)
    n = keys.shape[0]
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    c0 = keys.astype(np.uint64)
    c1 = np.full(n, frame & 0xFFFFFFFF, np.uint64)
    c2 = np.full(n, group & 0xFFFFFFFF, np.uint64)
    c3 = np.zeros(n, np.uint64)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & M, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & M
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return (c0 >> np.uint64(8)).astype(np.uint32)


@functools.lru_cache(maxsize=None)
def key_table(seed, fidx, group):
    return philox_u24(seed, np.arange(KEYS, dtype=np.uint64), fidx, group)


def pick_key(seed, fidx, group, lo, hi, taken, grid=False):
    """A row key whose uniform lies in [lo, hi) (and is a multiple of 1/64 with grid=True), not in `taken`."""
    U = key_table(seed, fidx, group)
    a, b = math.ceil(lo * 2 ** 24), math.ceil(hi * 2 ** 24)
    ok = (U >= a) & (U < b)
    if grid:
        ok &= (U & np.uint32((1 << 18) - 1)) == 0
    for k in np.flatnonzero(ok):
        if int(k) not in taken:
            taken.add(int(k))
            return int(k)
    raise AssertionError(f"no row key with u in [{lo}, {hi}) grid={grid} among {KEYS} (seed {seed}, frame {fidx}, group {group})")


# ================================================================================================ fp64 reference
def fast_path_route(s, k):
    """Replay of sample_fast's bin arithmetic on processed fp32 scores: (route, threshold bin, its count, kept count)."""
    s = np.asarray(s, np.float32)
    fin = s > -np.inf
    mx = s[fin].max()
    lo = np.float32(mx - np.float32(32))
    x = (s[fin] - lo) * np.float32(64)
    bins = np.clip(x, 0, 2047).astype(np.int64)
    hist = np.bincount(bins, minlength=2048)
    above = np.concatenate([np.cumsum(hist[::-1])[::-1][1:], [0]])   # scores in higher bins
    tbs = np.flatnonzero((above < k) & (k <= above + hist))
    if not len(tbs):
        return "fewer_finite", -1, 0, 0
    tb = int(tbs[0])
    nc = int(hist[tb])
    if nc > 256:
        return "bin_overflow", tb, nc, 0
    cand = np.sort(s[fin][bins == tb])[::-1]
    thr = cand[k - int(above[tb]) - 1]
    m = int((s[fin] >= thr).sum())
    return ("kept_overflow" if m > 384 else "fast"), tb, nc, m


def exp_terms(s):
    """fp64 p_i = exp(fl32(s_i - max)) over token ids (0 for -inf) and the per-term error bound eps_i * p_i."""
    s = np.asarray(s, np.float32)
    fin = s > -np.inf
    d = np.where(fin, s - s[fin].max(), np.float32(0)).astype(np.float32)
    p = np.where(fin, np.exp(d.astype(np.float64)), 0.0)
    eps = np.where(fin & (d != 0), (3 + np.floor(1.173 * np.abs(d.astype(np.float64)))) * 2.0 ** -23, 0.0)
    return p, eps * p, fin


def error_budget(s):
    """(p, C, T, E, m, exact): fp64 probabilities and CDF of processed scores, and the fp32 error budget E (0 when every
    kept p is exactly 1, i.e. all kept scores are equal)."""
    p, ep, fin = exp_terms(s)
    C = np.cumsum(p)
    T = float(C[-1])
    m = int(fin.sum())
    exact = bool(ep.sum() == 0 and np.all(p[fin] == 1.0))
    E = 0.0 if exact else float(ep.sum() + (m - 1) * 2.0 ** -24 * T + m * 2.0 ** -126)
    return p, C, T, E, m, exact


def cdf_token(p, C, u):
    t = u * C[-1]
    j = int(np.searchsorted(C, t, side="right"))
    j = min(j, len(C) - 1)
    while p[j] == 0 and j > 0:
        j -= 1
    return j


def cdf_agrees(s, u, tok):
    """True if `tok` is the inverse-CDF token of u or every CDF boundary between the two lies within the bound.
    Returns (ok, exact_token, near) where near says the draw needed the bound."""
    p, C, T, E, m, exact = error_budget(s)
    want = cdf_token(p, C, u)
    if tok == want:
        return True, want, False
    tgt = u * T
    tgt_exact = float(np.float32(u) * np.float32(T)) == tgt
    bound = (1 + u) * E + (0.0 if tgt_exact else 2.0 ** -24 * u * T)
    lo, hi = min(tok, want), max(tok, want)
    # a zero bound (grid rows, exact target) decides the draw exactly: a boundary equal to u * T is no tolerance
    ok = bound > 0 and bool(np.all(np.abs(C[lo:hi] - tgt) <= bound * 1.0001)) and p[tok] > 0
    return ok, want, True


def topp_sets(s_topk, top_p):
    """Kept / ambiguous token sets of top-p applied to the top-k scores: (kept, ambiguous) boolean arrays."""
    s = np.asarray(s_topk, np.float32)
    p, C, T, E, m, exact = error_budget(s)
    order = np.argsort(s, kind="stable")
    fin = s > -np.inf
    share = np.zeros(len(s))
    share[order] = np.cumsum(p[order]) / T
    thr_k = float(np.float32(1.0) - np.float32(top_p))
    thr_o = float(np.float32(1.0 - top_p))
    slack = 0.0 if (exact and m & (m - 1) == 0) else 2 * E / T + 2.0 ** -23
    lo, hi = min(thr_k, thr_o) - slack, max(thr_k, thr_o) + slack
    top = np.zeros(len(s), bool)
    top[order[-1]] = True
    kept = fin & (top | (share > hi))
    amb = fin & ~kept & ((share > lo) if slack == 0 else (share >= lo))
    return kept, amb


def bf16_bits(x):
    return torch.as_tensor(np.asarray(x, np.float32)).bfloat16().view(torch.int16).numpy()


def bf16_val(x):
    return torch.as_tensor(np.asarray(x, np.float32)).bfloat16().float().numpy()


# ================================================================================================ launches
@dataclass
class Launch:
    name: str
    group: int                      # 0 talker, 1..G-1 code-predictor codebook
    logits: np.ndarray              # [B][V] fp32
    do_sample: int = 1
    top_k: int = 50
    top_p: float = 1.0
    temperature: float = 1.0
    rp: float = 1.0
    min_new: int = 0
    suppress_eos: int = 0
    seed: int = 7
    frame: int = 3
    in_prefill: int = 0
    admit_mask: int = 0xFFFFFFFF
    seen: list = None               # per row: list of seen ids
    n_gen: list = None
    finished: list = None
    frame0: list = None
    aims: list = None               # per row: None | ("u", lo, hi) | ("tok", ids) | ("grid",)
    forced: list = None             # per row: forced token for this fidx (-1 none); None disables teacher forcing
    trailing_len: list = None
    keys: list = None               # filled by finish()
    tags: set = field(default_factory=set)

    @property
    def B(self):
        return self.logits.shape[0]

    @property
    def V(self):
        return self.logits.shape[1]

    def fidx(self, b):
        f = self.frame - self.frame0[b]
        return (0 if self.in_prefill else f + 1) if self.group == 0 else f


def processed(L, b):
    """Oracle scores of row b (HF processors, oracle/sampler.py)."""
    lg = L.logits[b]
    if L.group == 0:
        seen = sorted(L.seen[b])
        n = L.n_gen[b]
        assert n >= len(seen)
        gen = (seen + [seen[0]] * (n - len(seen))) if seen else [0] * n
        mn = n + 1 if L.suppress_eos else L.min_new
        return OS.process_logits(lg, generated_ids=gen, repetition_penalty=L.rp if seen else 1.0, min_new_tokens=mn,
                                 eos_token_id=EOS, suppress_lo=L.V - 1024, suppress_hi=L.V, do_sample=bool(L.do_sample),
                                 temperature=L.temperature, top_k=L.top_k, top_p=L.top_p)
    return OS.process_logits(lg, do_sample=bool(L.do_sample), temperature=L.temperature, top_k=L.top_k, top_p=L.top_p)


def finish(L):
    """Fill per-row defaults and choose each row's Philox key from its aim."""
    B = L.B
    L.seen = L.seen or [[] for _ in range(B)]
    L.n_gen = L.n_gen or [len(s) + 3 for s in L.seen]
    L.finished = L.finished or [0] * B
    L.frame0 = L.frame0 or [0] * B
    L.aims = L.aims or [None] * B
    L.trailing_len = L.trailing_len or [2] * B
    taken, keys = set(), []
    for b in range(B):
        a, f = L.aims[b], L.fidx(b)
        if a is None:
            keys.append(1000 + 37 * b)
            continue
        if a[0] == "grid":
            keys.append(pick_key(L.seed, f, L.group, 0.0, 1.0, taken, grid=True))
            continue
        if a[0] == "tok":
            s = processed(L, b)
            p, Cdf, T, _, _, _ = error_budget(s)
            ids = sorted(a[1])
            lo, hi = (Cdf[ids[0] - 1] if ids[0] else 0.0) / T, Cdf[ids[-1]] / T
            w = hi - lo
            assert w > 1e-5, (L.name, b, w)
            a = ("u", lo + 0.1 * w, hi - 0.1 * w)
        keys.append(pick_key(L.seed, f, L.group, a[1], a[2], taken))
    L.keys = keys
    return L


# ================================================================================================ shim
@pytest.fixture(scope="session")
def shim(tmp_path_factory):
    """tests/csrc/sampler_shim.cu compiled for sm_90a with the library's flags; it links against nothing."""
    from qwen3_tts_b200 import build
    out = str(tmp_path_factory.mktemp("sampler_shim") / "libsampler_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-shared", "-I", build.CSRC, SHIM_SRC, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"shim build failed:\n{r.stdout}\n{r.stderr}"
    lib = C.CDLL(out)
    vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
    lib.sampler_shim_layout.restype = C.c_longlong
    lib.sampler_shim_layout.argtypes = [C.c_char_p]
    lib.sampler_shim_run.restype = i32
    lib.sampler_shim_run.argtypes = ([i32] * 7 + [vp, vp, vp, C.POINTER(i32), C.POINTER(C.c_uint32), C.c_uint32,
                                                  C.POINTER(i32)] + [i32, i32, f32, f32, f32, i32, i32, f32, f32, i32, i32,
                                                                      C.c_ulonglong]
                                     + [vp] * 6 + [i32, vp, vp, i32, vp, vp, vp, i32, vp, i32, i32, i32, vp])
    lib.path = out
    lib.lay = {n: lib.sampler_shim_layout(n.encode()) for n in ("sizeof", "finished", "n_valid", "n_gen", "c0", "cur",
                                                                  "cur_stride", "max_batch", "max_vocab")}
    return lib


def guarded(rows, width, dtype, fill, dev, data=None):
    """[rows + 2][width] buffer with one guard row on each side; returns (buffer, pointer to row 1)."""
    buf = torch.full((rows + 2, width), fill, dtype=dtype, device=dev)
    if data is not None:
        buf[1:rows + 1] = data
    return buf, buf.data_ptr() + width * buf.element_size()


def tables(seed=5):
    """Embedding tables and inputs of the next-embed (bf16 values, fixed)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.5).bfloat16()  # noqa: E731
    return dict(emb_t=r(V_T, H), emb_cp=r((G - 1) * V_C, H), cp_next=r((G - 1) * V_C, WN), past=r(32, H),
                trailing=r(32, TS, H), pad=r(H), guard_t=r(2, H), guard_cp=r(2, H), guard_n=r(2, WN),
                cur=torch.randint(0, V_C, (32, G), generator=g, dtype=torch.int32))


TABLES = tables()


def run_launch(lib, L):
    """One shim launch of L; returns everything the phase may have written, on the host."""
    dev = "cuda"
    lay, B, V = lib.lay, L.B, L.V
    T = TABLES
    st = torch.zeros(lay["sizeof"], dtype=torch.uint8)
    sv = st.view(torch.int32)
    cur0 = T["cur"][:B].clone()

    def put(name, vals, stride=1):
        o = lay[name] // 4
        for b, v in enumerate(vals):
            sv[o + b * stride] = int(v)
    put("finished", L.finished)
    put("n_valid", [-7] * B)
    put("n_gen", L.n_gen)
    put("c0", [-5] * B)
    o = lay["cur"] // 4
    for b in range(B):
        sv[o + b * lay["cur_stride"]: o + b * lay["cur_stride"] + G] = cur0[b]
    st = st.to(dev)
    seen0 = torch.zeros(B, V_T, dtype=torch.uint8)
    for b in range(B):
        for t in L.seen[b]:
            seen0[b, t] = 1
    seen, seen_p = guarded(B, V_T, torch.uint8, SEEN_GUARD, dev, seen0)
    emb_t = torch.cat([T["guard_t"][:1], T["emb_t"], T["guard_t"][1:]]).to(dev)
    emb_cp = torch.cat([T["guard_cp"][:1], T["emb_cp"], T["guard_cp"][1:]]).to(dev)
    cp_next = torch.cat([T["guard_n"][:1], T["cp_next"], T["guard_n"][1:]]).to(dev)
    sent = lambda rows, w: guarded(rows, w, torch.int16, SENT_BF16, dev)  # noqa: E731
    x_cp, x_cp_p = sent(2 * B, H)
    nxt, nxt_p = sent(B, WN)
    th, th_p = sent(B, H)
    codes, codes_p = guarded(B, CS * G, torch.int32, SENT_CODE, dev)
    past = T["past"][:B].contiguous().to(dev)
    trailing = T["trailing"][:B].contiguous().to(dev)
    pad = T["pad"].to(dev)
    lg = torch.from_numpy(np.ascontiguousarray(L.logits, np.float32)).to(dev)
    forced = n_forced = None
    if L.forced is not None:
        n_forced = max(L.fidx(b) for b in range(B)) + 1
        fz = torch.full((B, n_forced, G), -1, dtype=torch.int32)
        for b in range(B):
            fz[b, L.fidx(b), L.group] = L.forced[b]
        forced = fz.to(dev)
    ia = lambda v: (C.c_int * B)(*v)  # noqa: E731
    talker = L.group == 0
    other = dict(do=0 if L.do_sample else 1, k=1, p=0.5, t=2.5)   # the other stack's fields differ from this one's
    sp = [L.do_sample, L.top_k, L.top_p, L.temperature] if talker else [other["do"], other["k"], other["p"], other["t"]]
    ssp = [other["do"], other["k"], other["p"], other["t"]] if talker else [L.do_sample, L.top_k, L.top_p, L.temperature]
    rc = lib.sampler_shim_run(L.group, B, V_T, V_C, H, G, EOS, lg.data_ptr() if talker else None,
                              None if talker else lg.data_ptr(), st.data_ptr(), ia(L.frame0),
                              (C.c_uint32 * B)(*L.keys), L.admit_mask, ia(L.trailing_len),
                              sp[0], sp[1], sp[2], sp[3], L.rp, ssp[0], ssp[1], ssp[2], ssp[3], L.min_new,
                              L.suppress_eos, L.seed, seen_p, emb_t.data_ptr() + H * 2, emb_cp.data_ptr() + H * 2,
                              x_cp_p, cp_next.data_ptr() + WN * 2, nxt_p, WN, past.data_ptr(), trailing.data_ptr(), TS,
                              pad.data_ptr(), th_p, codes_p, CS, None if forced is None else forced.data_ptr(),
                              n_forced or 0, L.frame, L.in_prefill, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, f"{L.name}: shim launch failed ({rc})"
    torch.cuda.synchronize()
    stc = st.cpu().view(torch.int32)

    def get(name, stride=1):
        o = lay[name] // 4
        return [int(stc[o + b * stride]) for b in range(B)]
    curv = torch.stack([stc[o + b * lay["cur_stride"]: o + b * lay["cur_stride"] + G] for b in range(B)])
    return dict(finished=get("finished"), n_valid=get("n_valid"), n_gen=get("n_gen"), c0=get("c0"), cur=curv.numpy(),
                cur0=cur0.numpy(), seen=seen.cpu(), seen0=seen0, x_cp=x_cp.cpu(), nxt=nxt.cpu(), th=th.cpu(),
                codes=codes.cpu(), tables_same=bool(torch.equal(emb_t[1:-1].cpu(), T["emb_t"])
                                                    and torch.equal(emb_cp[1:-1].cpu(), T["emb_cp"])
                                                    and torch.equal(cp_next[1:-1].cpu(), T["cp_next"])
                                                    and torch.equal(emb_t[[0, -1]].cpu(), T["guard_t"])
                                                    and torch.equal(emb_cp[[0, -1]].cpu(), T["guard_cp"])
                                                    and torch.equal(cp_next[[0, -1]].cpu(), T["guard_n"])))


def check_token(L, b, tok):
    """The rule of the module docstring for row b's freshly sampled token; returns a description on failure."""
    s = processed(L, b)
    if not L.do_sample:
        want = int(np.argmax(s))
        return None if tok == want else f"greedy: got {tok}, want {want}"
    u = philox.uniform(L.seed, L.keys[b], L.fidx(b), L.group)
    if L.aims[b] and L.aims[b][0] == "grid":
        STATS["grid_draws"] += 1
    pre = None
    if L.top_p < 1.0:
        pre = processed(Launch(L.name, L.group, L.logits, do_sample=1, top_k=L.top_k, temperature=L.temperature,
                               rp=L.rp, min_new=L.min_new, suppress_eos=L.suppress_eos, seen=L.seen, n_gen=L.n_gen), b)
    return sampled_token_error(s, pre, L.top_p, u, tok)


def sampled_token_error(s, s_pre_topp, top_p, u, tok):
    """The module docstring's rule for one sampled token: s = the oracle's processed scores, s_pre_topp = the same
    processing without top-p (when top_p < 1).  Returns None, or what is wrong."""
    STATS["sampled"] += 1
    if not (0 <= tok < len(s)):
        return f"token {tok} out of range"
    fin = s > -np.inf
    if top_p < 1.0:
        kept, amb = topp_sets(s_pre_topp, top_p)
        bad = (kept != fin) & ~amb
        assert not bad.any(), f"the oracle's top-p set differs from fp64 outside the bound at {np.flatnonzero(bad)[:5]}"
        if amb.any():   # either side of the bound may keep each ambiguous token: the draw must fit one resolution
            STATS["topp_ambiguous"] += 1
            ids = np.flatnonzero(amb)
            if not (fin[tok] or amb[tok]):
                return f"token {tok} outside the top-p kept set"
            if len(ids) > 6:
                return None
            for mask in range(1 << len(ids)):
                keep = kept.copy()
                keep[ids[[(mask >> i) & 1 == 1 for i in range(len(ids))]]] = True
                if keep[tok] and cdf_agrees(np.where(keep, s_pre_topp, np.float32(NEG)), u, tok)[0]:
                    return None
            return f"inverse CDF: token {tok} fits no resolution of the ambiguous top-p tokens {ids.tolist()} (u={u})"
    if not fin[tok]:
        return f"token {tok} outside the oracle's kept set (score {s[tok]})"
    ok, want, near = cdf_agrees(s, u, tok)
    assert cdf_agrees(s, u, OS.sample_from_scores(s, do_sample=True, u=u)[0])[0], \
        "the oracle's own token is off the fp64 CDF beyond the bound"
    STATS["near_boundary"] += int(near and ok)
    return None if ok else f"inverse CDF: got {tok}, want {want} (u={u})"


def check_launch(lib, L):
    out = run_launch(lib, L)
    B, V, what = L.B, L.V, L.name
    assert out["tables_same"], f"{what}: a read-only table or its guard rows changed"
    seen = out["seen"]
    assert bool((seen[0] == SEEN_GUARD).all() and (seen[-1] == SEEN_GUARD).all()), f"{what}: seen guard row written"
    for name, buf, fill in (("x_cp", out["x_cp"], SENT_BF16), ("next cp row", out["nxt"], SENT_BF16),
                            ("talker input", out["th"], SENT_BF16), ("codes_out", out["codes"], SENT_CODE)):
        assert bool((buf[0] == fill).all() and (buf[-1] == fill).all()), f"{what}: {name} guard row written"
    talker = L.group == 0
    if talker:   # codebook 0 writes neither codes_out nor a code-predictor / talker next-input row
        for name in ("nxt", "th", "codes"):
            assert bool((out[name] == (SENT_CODE if name == "codes" else SENT_BF16)).all()), f"{what}: {name} written"
    toks = out["c0"] if talker else [int(out["cur"][b, L.group]) for b in range(B)]
    assert all(0 <= t < V for b, t in enumerate(toks) if not (L.in_prefill and not (L.admit_mask >> b) & 1)), \
        f"{what}: tokens out of [0, {V}): {toks}"
    T = TABLES
    for b in range(B):
        active = not (L.in_prefill and not (L.admit_mask >> b) & 1)
        fidx = L.fidx(b)
        fr = L.frame - L.frame0[b]
        tag = f"{what} row {b}"
        if not active:   # admission prefill: a running row keeps all of its state
            assert out["c0"][b] == -5 and out["n_gen"][b] == L.n_gen[b] and out["finished"][b] == L.finished[b], tag
            assert out["n_valid"][b] == -7 and (out["cur"][b] == out["cur0"][b]).all(), tag
            assert torch.equal(seen[b + 1], out["seen0"][b]), tag
            assert bool((out["x_cp"][1 + b] == SENT_BF16).all() and (out["x_cp"][1 + B + b] == SENT_BF16).all()), tag
            continue
        tok = toks[b]
        forced = L.forced[b] if (L.forced is not None and L.forced[b] >= 0) else None
        if talker and L.finished[b]:
            assert tok == EOS, f"{tag}: finished row got {tok}, want EOS"
        elif forced is not None:
            assert tok == forced, f"{tag}: teacher forcing ignored ({tok} != {forced})"
        else:
            err = check_token(L, b, tok)
            assert err is None, f"{tag}: {err}"
        cur = out["cur0"][b].copy()
        if talker:
            fin0 = L.finished[b]
            exp_fin = 1 if (fin0 or tok == EOS) else 0
            assert out["finished"][b] == exp_fin, f"{tag}: finished {out['finished'][b]} != {exp_fin}"
            assert out["n_valid"][b] == (fidx if (not fin0 and tok == EOS) else -7), f"{tag}: n_valid {out['n_valid'][b]}"
            assert out["n_gen"][b] == L.n_gen[b] + (0 if fin0 else 1), f"{tag}: n_gen {out['n_gen'][b]}"
            sw = out["seen0"][b].clone()
            if not fin0 and tok != EOS:
                sw[tok] = 1
            assert torch.equal(seen[b + 1], sw), f"{tag}: seen bitmap differs"
            cur[0] = tok
            assert (out["cur"][b] == cur).all(), f"{tag}: cur {out['cur'][b]} != {cur}"
            assert torch.equal(out["x_cp"][1 + B + b], T["emb_t"][tok].view(torch.int16)), f"{tag}: CP input row 1"
            assert torch.equal(out["x_cp"][1 + b], T["past"][b].view(torch.int16)), f"{tag}: CP input row 0 (past_hidden)"
            continue
        j = L.group
        cur[j] = tok
        assert (out["cur"][b] == cur).all(), f"{tag}: cur {out['cur'][b]} != {cur}"
        assert out["c0"][b] == -5 and out["n_gen"][b] == L.n_gen[b] and out["finished"][b] == L.finished[b], tag
        assert torch.equal(seen[b + 1], out["seen0"][b]), f"{tag}: code predictor wrote seen"
        crow = out["codes"][1 + b].view(CS, G)
        want = torch.full((CS, G), SENT_CODE, dtype=torch.int32)
        if 0 <= fr < CS:
            want[fr, j] = tok
            if j == 1:
                want[fr, 0] = int(out["cur0"][b][0])
        assert torch.equal(crow, want), f"{tag}: codes_out row {crow.tolist()}"
        if j < G - 1:
            assert torch.equal(out["nxt"][1 + b], T["cp_next"][(j - 1) * V_C + tok].view(torch.int16)), f"{tag}: next CP row"
            assert bool((out["th"][1 + b] == SENT_BF16).all()), f"{tag}: talker input written by codebook {j}"
        else:
            s = T["emb_t"][int(cur[0])].float().numpy().astype(np.float32)
            for g2 in range(1, G):
                s = (s + T["emb_cp"][(g2 - 1) * V_C + int(cur[g2])].float().numpy()).astype(np.float32)
            txt = T["trailing"][b, fr] if fr < L.trailing_len[b] else T["pad"]
            want_h = bf16_bits(bf16_val(s) + txt.float().numpy())
            got_h = out["th"][1 + b].numpy()
            assert (got_h == want_h).all(), f"{tag}: talker input differs at {np.flatnonzero(got_h != want_h)[:8]}"
            assert bool((out["nxt"][1 + b] == SENT_BF16).all()), f"{tag}: next CP row written by the last codebook"


# ================================================================================================ cases
def rng(seed):
    return np.random.default_rng(seed)


def normal_rows(B, V, seed, scale=2.0, shift=0.0):
    return (rng(seed).standard_normal((B, V)) * scale + shift).astype(np.float32)


def stack(group):
    return (0, V_T) if group == 0 else (group, V_C)


def fast_path_cases(group):
    """Rows built to reach every branch of sample_fast (k <= 128, top_p = 1) and its fallbacks."""
    g, V = stack(group)
    hi_ids = lambda n, start=5: list(range(start, start + n))  # noqa: E731 (ids below V - 1024: never suppressed)
    out = []
    # k-th score inside max - 32 (normal logits), with u aimed at the k-th token's interval
    lg = normal_rows(4, V, 11 + g)
    out.append(Launch(f"fast.inside.g{g}", g, lg, top_k=50, temperature=0.9))
    # k-th beyond max - 32: one score far above; bin 0 holds <= 256 (rest -inf) or > 256 candidates
    lg = np.full((2, V), NEG, np.float32)
    lg[:, 3] = 40.0
    lg[0, hi_ids(200, 10)] = rng(12).standard_normal(200).astype(np.float32)
    lg[1, :] = rng(13).standard_normal(V).astype(np.float32)
    lg[1, 3] = 40.0
    out.append(Launch(f"fast.bin0.g{g}", g, lg, top_k=50, aims=[("u", 0.0, 1.0), ("u", 0.0, 1.0)]))
    # threshold bin with exactly 256 and 257 candidates (distinct scores inside one 1/64-wide bin), ten scores above
    rows = []
    for nc in (256, 257):
        r = np.full(V, -10.0, np.float32)
        r[hi_ids(10, 1000)] = 10.0 - np.arange(10, dtype=np.float32) * 0.25
        ids = hi_ids(nc, 20)
        r[ids] = np.float32(5.0) + np.arange(nc, dtype=np.float32) * np.float32(2 ** -16)
        rows.append((r, ids))
    lg = np.stack([r for r, _ in rows])
    out.append(Launch(f"fast.tb256.g{g}", g, lg, top_k=110,
                      aims=[("tok", ids[nc - 100 - 5: nc - 100 + 5]) for (_, ids), nc in zip(rows, (256, 257))]))
    # ties at the threshold: 127 distinct above, 256 tied (kept set 383, the largest the fast path can see) or 300 tied
    rows, aims = [], []
    for t in (256, 300, 3):
        r = np.full(V, -3.0, np.float32)
        r[hi_ids(127, 600)] = 2.0 + np.arange(127, dtype=np.float32) * 0.01
        r[hi_ids(t, 10)] = 1.0
        rows.append(r)
        aims.append(("tok", hi_ids(t, 10)))
    out.append(Launch(f"fast.ties.g{g}", g, np.stack(rows), top_k=128, aims=aims))
    # the tied threshold below the maximum: HF keeps all ties (a '>' would drop them)
    r = np.full((1, V), -6.0, np.float32)
    r[0, 7] = 1.0
    r[0, hi_ids(5, 30)] = 0.0
    out.append(Launch(f"fast.tie_below_max.g{g}", g, r, top_k=3, aims=[("tok", hi_ids(5, 30))]))
    # fewer than k finite scores
    r = np.full((2, V), NEG, np.float32)
    r[0, hi_ids(30, 40)] = rng(14).standard_normal(30).astype(np.float32)
    r[1, 9] = 0.5
    out.append(Launch(f"fast.fewer_finite.g{g}", g, r, top_k=50, aims=[("u", 0.0, 1.0), ("u", 0.0, 1.0)]))
    # all scores equal (grid: every p is exactly 1), -0.0 tied with +0.0, ~1e4 one ulp apart
    eq = np.zeros((2, V), np.float32)
    z = np.full(V, -4.0, np.float32)
    z[hi_ids(8, 50)] = np.array([0.0, -0.0] * 4, np.float32)
    z[4] = 1.0
    big = np.full(V, 9000.0, np.float32)
    u1 = np.float32(10000.0)
    big[hi_ids(20, 70)] = np.nextafter(u1, np.float32(0), dtype=np.float32)
    big[hi_ids(20, 70)[::2]] = u1
    out.append(Launch(f"fast.equal.g{g}", g, eq, top_k=50, aims=[("grid",), ("u", 0.0, 1.0)]))
    out.append(Launch(f"fast.zeros.g{g}", g, np.stack([z, z]), top_k=4, aims=[("tok", hi_ids(8, 50)), ("tok", [4])]))
    out.append(Launch(f"fast.ulp.g{g}", g, np.stack([big, big]), top_k=15, aims=[("tok", hi_ids(20, 70)[:10]),
                                                                                ("tok", hi_ids(20, 70)[10:])]))
    return out


def topk_cases(group):
    g, V = stack(group)
    out = []
    for k in (1, 2, 50, 127, 128, 129, 500, V - 1, 0, V, V + 5):
        lg = normal_rows(4, V, 100 + k % 997 + g, scale=1.5)
        out.append(Launch(f"topk{k}.g{g}", g, lg, top_k=k, temperature=0.9,
                          aims=[None, ("u", 0.0, 0.02), ("u", 0.49, 0.51), ("u", 0.98, 1.0)]))
    # radix select on negative scores (fkey's sign mapping) with ties at the 200th score; grid rows of 64 equal scores
    r = np.full((2, V), -9.0, np.float32)
    r[:, 100:299] = -2.0 - np.arange(199, dtype=np.float32) * 0.001
    r[:, 400:410] = -2.5
    r[1] = np.where(r[1] == -9.0, np.float32(-9.0), r[1])
    out.append(Launch(f"radix.neg.g{g}", g, r, top_k=200, aims=[("tok", list(range(400, 410))), ("u", 0.0, 1.0)]))
    gr = np.full((3, V), NEG, np.float32)
    gr[0, 40:104] = -1.5
    gr[1, 40:104] = 3.0
    gr[1, 200:300] = -30.0   # removed by top-k 64 (the kept set is the 64 equal scores)
    gr[2, 500:564] = -0.0
    out.append(Launch(f"grid.radix.g{g}", g, gr[[0, 2]], top_k=200, aims=[("grid",)] * 2, seed=21))
    out.append(Launch(f"grid.fast.g{g}", g, gr, top_k=64, aims=[("grid",)] * 3, seed=22))
    out.append(Launch(f"grid.none.g{g}", g, gr[[0, 2]], top_k=0, aims=[("grid",)] * 2, seed=23))
    return out


def topp_cases(group):
    g, V = stack(group)
    out = []
    for p in (0.0, 0.3, 0.8, 0.95, 0.9999):
        for k in (0, 50):
            lg = normal_rows(3, V, 200 + int(p * 100) + k + g, scale=1.2)
            lg[2, [11, 12]] = lg[2].max() + 1.0   # tie for the top score (p = 0 keeps the highest id of the tie)
            out.append(Launch(f"topp{p}.k{k}.g{g}", g, lg, top_k=k, top_p=p, temperature=0.9,
                              aims=[("u", 0.0, 0.05), ("u", 0.3, 0.7), ("u", 0.95, 1.0)]))
    # top-p at exactly 1 - p: m equal scores, every share (i+1)/m exact
    gr = np.full((2, V), NEG, np.float32)
    gr[:, 60:68] = 1.0
    for p in (0.5, 0.75, 0.625):
        for k in (0, 50):
            out.append(Launch(f"topp.grid{p}.k{k}.g{g}", g, gr, top_k=k, top_p=p, aims=[("grid",), ("grid",)], seed=31 + k))
    return out


def processor_cases():
    V = V_T
    out = []
    # repetition penalty on seen tokens of both signs: greedy rows built so that each branch decides the argmax
    pos = np.full(V, -1.0, np.float32)
    pos[[10, 20]] = [2.0, 1.9]
    neg = np.full(V, -5.0, np.float32)
    neg[[10, 20]] = [-1.0, -1.1]
    for rp in (0.8, 1.05, 1.3):
        out.append(Launch(f"penalty{rp}.greedy", 0, np.stack([pos, neg, pos, neg]), do_sample=0, rp=rp,
                          seen=[[10], [10], [20], [20, 30]]))
        lg = normal_rows(4, V, 300 + int(rp * 100), scale=1.5)
        seen = [list(np.flatnonzero(lg[b, :2048] > 1.0)[:40]) + list(np.flatnonzero(lg[b, :2048] < -1.0)[:40])
                for b in range(4)]
        out.append(Launch(f"penalty{rp}.sampled", 0, lg, rp=rp, seen=[[int(t) for t in s] for s in seen], top_k=0,
                          aims=[("u", 0.0, 0.1), ("u", 0.45, 0.55), ("u", 0.9, 1.0), None]))
    # min_new_tokens at n_gen = min - 1 and = min, suppress_eos; EOS the largest raw logit
    e = np.full(V, -2.0, np.float32)
    e[EOS] = 5.0
    e[33] = 4.0
    out.append(Launch("min_new", 0, np.stack([e, e, e]), do_sample=0, min_new=5, seen=[[1], [1], []], n_gen=[4, 5, 0]))
    out.append(Launch("suppress_eos", 0, np.stack([e, e]), do_sample=0, min_new=2, suppress_eos=1, seen=[[1], []],
                      n_gen=[9, 0]))
    # suppress-range edges: the maximum at V-1025 (kept), V-1024, V-1 (suppressed) and EOS (kept)
    rows = []
    for t in (V - 1025, V - 1024, V - 1, EOS, V - 1023):
        r = np.full(V, -1.0, np.float32)
        r[t] = 3.0
        r[100] = 2.0
        rows.append(r)
    out.append(Launch("suppress_edges.greedy", 0, np.stack(rows), do_sample=0, seen=[[]] * 5, n_gen=[0] * 5))
    out.append(Launch("suppress_edges.sampled", 0, np.stack(rows), top_k=2, seen=[[]] * 5, n_gen=[0] * 5,
                      aims=[("tok", [V - 1025]), ("tok", [100]), ("tok", [100]), ("tok", [EOS]), ("tok", [100])]))
    for T in (0.02, 0.9, 1.0, 3.0):
        for g in (0, 5):
            Vg = stack(g)[1]
            lg = normal_rows(4, Vg, 400 + int(T * 10) + g, scale=2.0)
            out.append(Launch(f"temp{T}.g{g}", g, lg, temperature=T, top_k=50,
                              aims=[("u", 0.0, 0.1), ("u", 0.4, 0.6), ("u", 0.9, 1.0), None]))
            out.append(Launch(f"temp{T}.k0.g{g}", g, lg, temperature=T, top_k=0, aims=[("u", 0.2, 0.8)] * 4))
    # greedy: ties for the maximum resolve to the lowest id; temperature is ignored
    for g in (0, 3):
        Vg = stack(g)[1]
        lg = normal_rows(3, Vg, 500 + g)
        lg[0, [700, 90, 1500]] = 9.0
        lg[1, :] = 0.25
        lg[2, [5, 6]] = [7.0, 7.0]
        out.append(Launch(f"greedy.ties.g{g}", g, lg, do_sample=0, temperature=0.02, top_k=1))
    return out


def bookkeeping_cases():
    """B = 32 rows with mixed finished / frame0 / row keys, in frame and admission-prefill mode, teacher forcing, EOS
    sampled, and the code predictor's next-input rows at codebooks 1, 7 and 15 around the trailing-text switch."""
    out = []
    B = 32
    r = rng(600)
    base = normal_rows(B, V_T, 601, scale=1.5)
    base[5, EOS] = 30.0          # samples EOS
    base[9, EOS] = 30.0          # ... but min_new keeps it out
    fin = [1 if b % 5 == 2 else 0 for b in range(B)]
    frame0 = [int(r.integers(0, 3)) for _ in range(B)]
    seen = [[int(t) for t in r.choice(2048, size=int(r.integers(0, 6)), replace=False)] for _ in range(B)]
    n_gen = [len(s) + int(r.integers(0, 4)) for s in seen]
    n_gen[5], n_gen[9], seen[9] = 6, 0, []
    aims = [("u", 0.05, 0.95) if b % 3 else None for b in range(B)]
    forced = [-1] * B
    forced[7], forced[11], forced[12] = 123, EOS, 2047
    for prefill in (0, 1):
        mask = 0xA5A5F00F if prefill else 0xFFFFFFFF
        out.append(Launch(f"book.talker.prefill{prefill}", 0, base, top_k=40, temperature=0.9, rp=1.3, min_new=2,
                          seen=seen, n_gen=n_gen, finished=fin, frame0=frame0 if not prefill else None, aims=aims,
                          in_prefill=prefill, admit_mask=mask, forced=forced, frame=4))
    cpl = normal_rows(B, V_C, 602, scale=1.5)
    tl = [int(r.integers(0, 5)) for _ in range(B)]
    fr0 = [int(r.integers(0, 3)) for _ in range(B)]
    for b in range(B):   # frame - frame0 == trailing_len (tts_pad) and == trailing_len - 1 (last text row) on some rows
        if b % 4 == 0:
            tl[b] = 3 - fr0[b]
        elif b % 4 == 1:
            tl[b] = 3 - fr0[b] + 1
    for j in (1, 7, G - 1):
        out.append(Launch(f"book.cp{j}", j, cpl, top_k=50, temperature=0.9, frame=3, frame0=fr0, trailing_len=tl,
                          finished=fin, aims=aims, forced=[-1] * 3 + [17] + [-1] * (B - 4)))
        out.append(Launch(f"book.cp{j}.greedy", j, cpl, do_sample=0, frame=8, frame0=fr0, trailing_len=tl))
    return out


def all_cases():
    cs = []
    for g in (0, 1):
        cs += fast_path_cases(g) + topk_cases(g) + topp_cases(g)
    cs += processor_cases() + bookkeeping_cases()
    return [finish(L) for L in cs]


@functools.lru_cache(maxsize=None)
def cases():
    return all_cases()


# ================================================================================================ CPU tests
def test_numpy_philox_matches_oracle():
    keys = np.array([0, 1, 2, 77, 2 ** 31 + 5, 2 ** 32 - 1], dtype=np.uint64)
    for seed, fr, grp in ((0, 0, 0), (7, 3, 1), (2 ** 40 + 3, 11, 15)):
        got = philox_u24(seed, keys, fr, grp)
        for k, v in zip(keys, got):
            assert float(v) / 2 ** 24 == philox.uniform(seed, int(k), fr, grp)


def test_reference_bound_and_top_p_sets():
    """The fp64 CDF token matches the oracle's on well-separated draws; grid rows have a zero budget; the top-p sets of
    a grid row at exactly 1 - p are exact."""
    s = np.full(16, NEG, np.float32)
    s[4:8] = 2.0
    p, Cdf, T, E, m, exact = error_budget(s)
    assert exact and E == 0 and T == 4 and m == 4
    assert cdf_token(p, Cdf, 0.5) == 6 and cdf_token(p, Cdf, 0.0) == 4 and cdf_token(p, Cdf, 0.75) == 7
    kept, amb = topp_sets(s, 0.5)
    assert not amb.any() and list(np.flatnonzero(kept)) == [6, 7]
    kept, amb = topp_sets(s, 0.0)
    assert list(np.flatnonzero(kept)) == [7]
    x = normal_rows(1, 300, 1)[0]
    p, Cdf, T, E, m, exact = error_budget(x)
    assert not exact and 0 < E < 1e-4 * T
    for u in (0.1, 0.5, 0.9):
        assert cdf_agrees(x, u, OS.sample_from_scores(x, do_sample=True, u=u)[0])[0]


def test_cases_reach_every_fast_path_branch():
    """Replaying sample_fast's bins on the processed scores: the case list reaches each branch.  The kept-set overflow
    (m > 384) cannot be reached: m <= (k - 1) + 256 = 383, since every kept score is in a higher bin or among the <= 256
    candidates of the threshold bin; the largest reachable kept set (383) is a case."""
    seen = set()
    for L in cases():
        if not L.do_sample or not (L.top_p >= 1.0 and 0 < L.top_k < L.V and L.top_k <= 128):
            continue
        for b in range(L.B):
            route, tb, nc, m = fast_path_route(processed(Launch(L.name, L.group, L.logits, do_sample=1, top_k=0,
                                                                temperature=L.temperature, rp=L.rp, min_new=L.min_new,
                                                                suppress_eos=L.suppress_eos, seen=L.seen, n_gen=L.n_gen), b),
                                               L.top_k)
            seen.add(route)
            if route == "fast":
                seen.add("kth_inside" if tb > 0 else "kth_in_bin0")
                seen.add(f"nc{nc}" if nc in (256,) else "")
                seen.add("m383" if m == 383 else "")
                assert m <= L.top_k - 1 + 256
            if route == "bin_overflow":
                seen.add("bin0_overflow" if tb == 0 else f"nc{nc}" if nc == 257 else "tie_overflow")
    want = {"fast", "fewer_finite", "bin_overflow", "kth_inside", "kth_in_bin0", "bin0_overflow", "nc256", "nc257",
            "tie_overflow", "m383"}
    assert want <= seen, want - seen


def test_shim_builds_and_exports_the_state_layout(shim):
    """The shim cross-compiles for sm_90a, defines only its own entry points, and exports the DevState layout."""
    syms = subprocess.run(["nm", "-D", shim.path], capture_output=True, text=True).stdout.splitlines()
    defined = [ln.split()[-1] for ln in syms if len(ln.split()) == 3 and ln.split()[1] in "TtDdBbRr"]
    undefined = [ln.split()[-1] for ln in syms if len(ln.split()) == 2 and ln.split()[0] == "U"]
    assert {"sampler_shim_run", "sampler_shim_layout"} <= set(defined)
    assert not [s for s in defined + undefined if "q3_" in s or "gemm_" in s], (defined, undefined)
    lay = shim.lay
    assert lay["max_batch"] == 32 and lay["max_vocab"] >= V_T and lay["cur_stride"] >= G
    assert all(lay[n] % 4 == 0 and 0 < lay[n] < lay["sizeof"] for n in ("finished", "n_valid", "n_gen", "c0", "cur"))


# ================================================================================================ GPU tests
@pytest.fixture(scope="module")
def lib(shim):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    yield shim
    print(f"\nsampler draws: {STATS['sampled']} sampled, {STATS['grid_draws']} exact grid draws, {STATS['near_boundary']} "
          f"inside the CDF bound, {STATS['topp_ambiguous']} rows with a top-p share inside its bound")


GROUPS = {
    "fast_path": lambda L: L.name.startswith("fast."),
    "top_k": lambda L: L.name.startswith(("topk", "radix", "grid")),
    "top_p": lambda L: L.name.startswith("topp"),
    "processors": lambda L: L.name.startswith(("penalty", "min_new", "suppress", "temp", "greedy")),
    "bookkeeping": lambda L: L.name.startswith("book."),
}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(GROUPS))
def test_sample_phase_against_oracle(lib, kind):
    sel = [L for L in cases() if GROUPS[kind](L)]
    assert sel
    for L in sel:
        check_launch(lib, L)


def test_every_case_is_in_a_group():
    assert all(any(f(L) for f in GROUPS.values()) for L in cases())


@pytest.mark.gpu
def test_invalid_sampling_parameters_are_rejected_before_any_launch():
    """q3_prefill / q3_session_begin reject sampling parameters the sample phase cannot handle and name the field.  Every
    call also passes an invalid batch (B = 0, n_slots = 0), so a library without the check fails on the batch instead
    and nothing is ever launched with these parameters."""
    from oracle import talker as OT
    from qwen3_tts_b200 import _lib
    from qwen3_tts_b200.engine import AREngine
    from tests import helpers as Hh
    cfg = OT.cfg_tiny()
    Wb, _ = Hh.bf16_weights(OT.random_weights(cfg, seed=1))
    eng = AREngine(Hh.to_pkg_cfg(cfg), Wb, device="cuda:0", max_batch=4, max_ctx=64)
    good = Hh.to_pkg_sampling(OT.SamplingCfg())
    H = cfg.talker.hidden_size
    pad = torch.zeros(H, dtype=torch.bfloat16, device="cuda:0")
    emb = torch.zeros(4, H, dtype=torch.bfloat16, device="cuda:0")
    lens = (C.c_int32 * 1)(4)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    nan, inf = float("nan"), float("inf")
    bad = [("temperature", dict(temperature=0.0)), ("temperature", dict(temperature=-1.0)),
           ("temperature", dict(temperature=nan)), ("temperature", dict(temperature=inf)),
           ("subtalker_temperature", dict(subtalker_temperature=0.0)),
           ("subtalker_temperature", dict(subtalker_temperature=-inf)),
           ("top_k", dict(top_k=-1)), ("subtalker_top_k", dict(subtalker_top_k=-3)),
           ("top_p", dict(top_p=-0.1)), ("top_p", dict(top_p=1.5)), ("top_p", dict(top_p=nan)),
           ("subtalker_top_p", dict(subtalker_top_p=nan)), ("subtalker_top_p", dict(subtalker_top_p=2.0)),
           ("repetition_penalty", dict(repetition_penalty=0.0)), ("repetition_penalty", dict(repetition_penalty=nan)),
           ("repetition_penalty", dict(repetition_penalty=-1.0)), ("repetition_penalty", dict(repetition_penalty=inf)),
           ("min_new_tokens", dict(min_new_tokens=-1))]
    for field_name, kw in bad:
        s = eng._sampling(good)
        for k, v in kw.items():
            setattr(s, k, v)
        rc = eng.lib.q3_prefill(eng.h, 0, emb.data_ptr(), lens, None, lens, 0, pad.data_ptr(), C.byref(s), stream)
        msg = eng.lib.q3_last_error().decode()
        assert rc != 0 and field_name in msg, (field_name, kw, rc, msg)
        rc = eng.lib.q3_session_begin(eng.h, 0, 0, pad.data_ptr(), C.byref(s), stream)
        msg = eng.lib.q3_last_error().decode()
        assert rc != 0 and field_name in msg, ("session", field_name, kw, rc, msg)
    # greedy ignores its temperature: do_sample = 0 with temperature 0 passes the check (and then fails on B = 0)
    s = eng._sampling(good)
    s.do_sample, s.temperature, s.subtalker_dosample, s.subtalker_temperature = 0, 0.0, 0, -1.0
    rc = eng.lib.q3_prefill(eng.h, 0, emb.data_ptr(), lens, None, lens, 0, pad.data_ptr(), C.byref(s), stream)
    assert rc != 0 and "batch" in eng.lib.q3_last_error().decode()
    with pytest.raises(RuntimeError, match="top_k"):
        s = eng._sampling(good)
        s.top_k = -1
        _lib.check(eng.lib.q3_session_begin(eng.h, 0, 0, pad.data_ptr(), C.byref(s), stream))
    torch.cuda.synchronize()
    eng.close()
