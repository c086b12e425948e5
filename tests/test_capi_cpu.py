"""CPU tests of the C-ABI library: it builds for sm_90a, loads, exports every symbol include/hhg.h
declares, and refuses to run without a GPU (no CPU fallback)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_match_header(hhg):
    lib = hhg.capi.load()
    hdr = open(os.path.join(ROOT, "include", "hhg.h")).read()
    declared = set(re.findall(r"\b(hhg_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    assert set(hhg.capi.SYMBOLS) <= declared


def test_sass_is_sm90a_only():
    import subprocess
    so = os.path.join(ROOT, "hh-suite_b200", "libhhg.so")
    out = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="GPU present")
def test_no_cpu_fallback(hhg):
    with pytest.raises(hhg.HhgError) as e:
        hhg.Context()
    assert "no CPU fallback" in str(e.value)
