"""C-ABI checks that need no GPU: the library loads, exports every symbol include/rnnoise.h declares,
parses/rejects model blobs like the reference's parser, and refuses to run without a CUDA device
(there is no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from rnnoise_b200 import build
    build.build()
    import rnnoise_b200
    return rnnoise_b200.lib()


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "rnnoise.h")).read()
    return sorted(set(re.findall(r"RNNOISE_EXPORT[^;(]*?\b(rnnoise_\w+)\s*\(", hdr)))


def test_every_declared_symbol_is_exported(L):
    syms = declared_symbols()
    assert len(syms) >= 20 and "rnnoise_process_frame_batch" in syms and "rnnoise_create" in syms
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/rnnoise.h but not exported"


def test_only_public_symbols_are_exported():
    import subprocess
    import rnnoise_b200
    out = subprocess.run(["nm", "-D", "--defined-only", rnnoise_b200.LIB_PATH], capture_output=True, text=True).stdout
    names = [l.split()[-1] for l in out.splitlines() if " T " in l]
    assert names and all(n.startswith("rnnoise_") for n in names), names


def test_sizes(L):
    assert L.rnnoise_get_frame_size() == 480
    assert L.rnnoise_get_size() > 0


def test_model_parse_and_reject(L, models_dir):
    for name in ("default", "hot", "little", "g256", "tiny"):
        m = L.rnnoise_model_from_filename(os.path.join(models_dir, name + ".bin").encode())
        assert m
        L.rnnoise_model_free(m)
    assert not L.rnnoise_model_from_filename(b"/nonexistent/blob.bin")   # reference would crash here
    blob = open(os.path.join(models_dir, "default.bin"), "rb").read()
    assert not L.rnnoise_model_from_buffer(blob, len(blob) - 100)
    assert not L.rnnoise_model_from_buffer(blob[64:], len(blob) - 64)
    # drop one record (first array) -> a required array is missing -> rejected like linear_init does
    first = 64 + int.from_bytes(blob[16:20], "little")
    assert not L.rnnoise_model_from_buffer(blob[first:], len(blob) - first)
    m = L.rnnoise_model_from_buffer(blob, len(blob))
    assert m
    L.rnnoise_model_free(m)


def test_no_cpu_fallback(L, models_dir):
    """Without a CUDA device every creation entry point must fail loudly instead of computing on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    m = L.rnnoise_model_from_filename(os.path.join(models_dir, "default.bin").encode())
    assert not L.rnnoise_batch_create(m, 4, 0)
    assert not L.rnnoise_create(m)
    L.rnnoise_model_free(m)


def test_product_does_not_reference_oracle():
    """The product tree must not import, link or include anything under oracle/."""
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "rnnoise_b200")):
        for f in files:
            if f.endswith((".c", ".cu", ".cuh", ".h", ".hpp", ".py")):
                txt = open(os.path.join(d, f), errors="ignore").read()
                if re.search(r"(#include|import|from)\s+[\"<]?\.*/?oracle", txt) or "rnnoise_port" in txt.replace("oracle/rnnoise_port.c is the executable statement", ""):
                    bad.append(f)
    assert not bad, bad


def test_reference_demo_links_unchanged(tmp_path):
    """examples/rnnoise_demo.c of the reference compiles and links against our header + library
    unmodified.  Needs the reference sources where oracle/build_ref.py looks for them ($RNNOISE_REFERENCE); skipped
    where they are absent, because no reference source may be stored in this repository."""
    import subprocess
    import rnnoise_b200
    from oracle.build_ref import REF
    demo = os.path.join(REF, "examples", "rnnoise_demo.c")
    if not os.path.exists(demo):
        pytest.skip("reference tree not present")
    exe = str(tmp_path / "rnnoise_demo")
    r = subprocess.run(["gcc", "-DUSE_WEIGHTS_FILE", "-I", os.path.join(ROOT, "include"), demo, "-o", exe,
                        rnnoise_b200.LIB_PATH, "-Wl,-rpath," + os.path.dirname(rnnoise_b200.LIB_PATH)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_batch_demo_compiles_links_and_fails_cleanly_without_gpu(tmp_path, models_dir):
    """examples/rnnoise_batch_demo.c (multi-file denoiser over the multi-frame int16 call) builds against the
    public header + library with a plain C compiler; without a GPU it must stop with the no-CPU-path message,
    not crash."""
    import subprocess
    import numpy as np
    import rnnoise_b200
    exe = str(tmp_path / "rnnoise_batch_demo")
    r = subprocess.run(["gcc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "rnnoise_batch_demo.c"),
                        "-o", exe, rnnoise_b200.LIB_PATH, "-Wl,-rpath," + os.path.dirname(rnnoise_b200.LIB_PATH)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = str(tmp_path / "a.raw")
    (np.arange(2000) % 100).astype(np.int16).tofile(raw)
    r = subprocess.run([exe, os.path.join(models_dir, "tiny.bin"), raw], capture_output=True, text=True)
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        assert r.returncode == 0 and os.path.getsize(raw + ".denoised") == 5 * 480 * 2, r.stderr
    else:
        assert r.returncode == 1 and "no CPU path" in r.stderr, (r.returncode, r.stderr)
