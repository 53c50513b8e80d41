"""CPU model of the tap-GEMM kernel's tiling (csrc/gemm_sm90.cu): the accumulator-fragment index math the epilogue uses
to find each output element, and the shared-memory budget of every tile width.  The constants are read from the CUDA
source so the model follows the kernel."""
import os
import re

SRC = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "qwen3-tts_b200", "csrc", "gemm_sm90.cu")).read()
TILE_WIDTHS = (64, 128)   # what gemm_make_plan_v accepts


def const(name):
    m = re.search(rf"constexpr int {name} = ([^;]+);", SRC)
    assert m, name
    expr = m.group(1).split("//")[0]
    return int(eval(expr, {}, {k: const(k) for k in re.findall(r"[A-Z_]{2,}", expr) if k != name}))


def fragment(warp, lane, i):
    """(row, column) inside a warpgroup's 64 x bn accumulator of accumulator register i (m64nNk16, f32)"""
    j, h, e = i // 4, (i // 2) % 2, i % 2
    return 16 * (warp % 4) + lane // 4 + 8 * h, 8 * j + 2 * (lane % 4) + e


def test_fragments_cover_each_warpgroup_tile_exactly_once():
    for bn in TILE_WIDTHS:
        seen = {}
        for warp in range(4):
            for lane in range(32):
                for i in range(bn // 2):
                    rc = fragment(warp, lane, i)
                    assert rc not in seen, (bn, rc)
                    seen[rc] = (warp, lane, i)
        assert sorted(seen) == [(r, c) for r in range(64) for c in range(bn)]


def test_pair_and_gated_epilogues_read_matching_columns():
    for bn in TILE_WIDTHS:
        for warp in range(4):
            for lane in range(32):
                for j in range(bn // 8):
                    for h in range(2):
                        r0, c0 = fragment(warp, lane, 4 * j + 2 * h)
                        r1, c1 = fragment(warp, lane, 4 * j + 2 * h + 1)
                        assert r0 == r1 and c0 % 2 == 0 and c1 == c0 + 1   # one 4-byte bf16 pair per store
                for j in range(bn // 16):   # ACT_SWIGLU_BLK8: gate in columns 16j..16j+7, up 8 columns later, same row
                    for h in range(2):
                        for e in range(2):
                            rg, cg = fragment(warp, lane, 8 * j + 2 * h + e)
                            ru, cu = fragment(warp, lane, 8 * j + 4 + 2 * h + e)
                            assert rg == ru and cu == cg + 8 and cg // 16 == j and cg % 16 < 8


def test_shared_memory_budget_for_every_tile_width():
    BM, BK = const("BM"), const("BK")
    a_bytes = BM * BK * 2
    optin, bar, max_stages = const("SMEM_OPTIN"), const("BAR_BYTES"), const("MAX_STAGES")
    assert const("A_BYTES") == a_bytes and 2 * 8 * max_stages <= bar
    for bn in TILE_WIDTHS:
        stage = a_bytes + ((bn * BK * 2 + 1023) & ~1023)
        nst = min(max_stages, (optin - 1024 - bar) // stage)
        assert nst >= 4, (bn, nst)                      # the TMA ring never gets shallower than 4 stages
        assert 1024 + nst * stage + bar <= optin        # what gemm_launch asks for fits the 227 KB opt-in
        assert stage % 1024 == 0                        # SWIZZLE_128B operand tiles stay 1024-byte aligned
    threads = const("GEMM_THREADS")
    assert threads == 128 * const("CONSUMER_WGS") + 32 and const("PRODUCER_WARP") == 4 * const("CONSUMER_WGS")
    assert BM == 64 * const("CONSUMER_WGS")
