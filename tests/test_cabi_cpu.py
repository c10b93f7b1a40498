"""CPU tests of the boundary: the C-ABI library builds, loads and exports every symbol include/*.h declares;
without a GPU every compute entry fails loudly (no CPU fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "adaptive_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ac_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(cabi):
    L = cabi.load_library()
    declared = _header_functions()
    assert len(declared) >= 30
    for name in declared:
        assert hasattr(L, name), f"{name} declared in include/adaptive_b200.h but not exported"
    for name in cabi.EXPORTS:
        assert name in declared, f"{name} bound in _cabi.py but not declared in the header"
    assert L.ac_version() == 1


def test_header_cites_reference_call_sites():
    src = open(os.path.join(ROOT, "include", "adaptive_b200.h")).read()
    for cite in ("memory.py:110-114", "models.py:71-80", "classifier.py:1271-1275", "ewc.py", "classifier.py:1358-1384"):
        assert cite in src


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback(cabi):
    L = cabi.load_library()
    assert L.ac_device_check() != 0
    assert b"no CPU fallback" in L.ac_last_error() or b"CUDA" in L.ac_last_error()
    import adaptive_classifier_b200 as acb
    with pytest.raises(acb.AdaptiveB200Error):
        acb.AdaptiveClassifier("bert-base-uncased")
    with pytest.raises(acb.AdaptiveB200Error):
        acb.AdaptiveClassifier("bert-base-uncased", device="cpu")
    head = acb.AdaptiveHead(16, 3, hidden_dims=[16, 8]).eval()
    with pytest.raises(acb.AdaptiveB200Error):
        head(torch.zeros(2, 16))
    mem = acb.PrototypeMemory(16)
    with pytest.raises(acb.AdaptiveB200Error):
        mem.add_example(acb.Example("t", "a", torch.zeros(16)), "a")


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "adaptive_classifier_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "oracle/" not in txt.replace("oracle/knn_oracle.c", "").replace("oracle/precision_study.py", "").replace("oracle/deferred_ln_study.py", ""), f   # comments citing the studies


def test_no_kernel_selector_switches_in_the_shipped_abi(cabi):
    """round 2: every kernel variant was either promoted to THE implementation or deleted; the library has no
    ac_set_option-style selectors and no environment switchboard"""
    L = cabi.load_library()
    assert not hasattr(L, "ac_set_option") and not hasattr(L, "ac_get_option")
    for name in _header_functions():
        assert "option" not in name and "peer" not in name


def test_head_training_kernel_on_the_cpu_emulation():
    """csrc/head_train.cuh (the persistent cooperative training kernel: ownership blocks, streamed chunks, six grid barriers per
    step) is plain SIMT C++; tests/cpu_shim runs it with every CUDA thread as a fiber and real grid barriers (thread order
    shuffled between barriers) and compares several optimizer steps / a gradient-only call with a natural-order restatement.
    This is how the kernel's logic was checked before any GPU time was spent on it."""
    import subprocess, tempfile
    shim = os.path.join(ROOT, "tests", "cpu_shim")
    exe = os.path.join(tempfile.mkdtemp(prefix="ht_emul_"), "head_train_emul")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-I/usr/local/cuda/include", os.path.join(shim, "head_train_emul.cpp"),
                        os.path.join(shim, "cuda_shim.cpp"), "-o", exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    #        D   H0  H1  C    n  batch G loss dropout ewc update seed [z_shift]
    cases = ["40 40 20 5 50 20 3 0 0.1 0 1 1",          # CE, dropout, last batch partial
             "40 40 20 5 50 20 2 1 0.1 0 1 2",          # BCE; 2 CTAs -> several ownership blocks per CTA
             "264 136 68 11 70 32 4 0 0.1 1 1 3",       # K not a multiple of the chunk width; EWC with a grown head
             "64 64 32 3 45 40 3 0 0.0 1 1 4",          # batch > 32 (two rows per lane), C = 3 (scalar chunk loads)
             "128 128 64 130 64 32 5 1 0.2 1 1 5",      # C > one chunk: dz streamed in two chunks
             "264 136 68 11 30 30 4 0 0.0 0 0 6",       # gradient-only mode (Fisher): gradients and accumulators
             "40 40 20 5 20 20 1 1 0.0 1 0 7",          # a single CTA owns everything
             "40 40 20 5 50 20 9 0 0.1 1 1 9",
             "264 136 68 11 70 32 28 0 0.1 1 1 10",
             "520 264 68 11 30 30 4 0 0.0 0 0 6",       # several 256-column chunks per product
             "128 128 64 130 64 32 5 0 0.2 1 1 11",     # CE with more than 128 classes (logit tail re-read)
             "520 264 68 11 40 3 4 0 0.1 0 0 12",       # partials of the row products larger than the ring they share (batch 3)
             "40 40 20 6 24 12 3 1 0.0 0 0 13 30"]      # BCE at saturated logits (z ~ +-30): ATen's vanishing gradient
    for c in cases:
        out = subprocess.run([exe] + c.split(), capture_output=True, text=True, timeout=600)
        assert out.returncode == 0 and "MATCH" in out.stdout, (c, out.stdout[-600:], out.stderr[-300:])
