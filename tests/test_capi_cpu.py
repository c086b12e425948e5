"""CPU tests of the C-ABI library: it builds for sm_90a, loads, exports every symbol include/hhg.h
declares, is bound with the header's own prototypes, mirrors the header's structs with the compiler's layout,
and refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "hhg.h")


def test_exports_match_header(hhg):
    lib = hhg.capi.load()
    hdr = open(HEADER).read()
    declared = set(re.findall(r"\b(hhg_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    assert set(hhg.capi.SYMBOLS) <= declared
    # the prototype parse that binds the library skips no declaration, and binds each one's signature
    assert declared <= set(hhg.capi.SYMBOLS), sorted(declared - set(hhg.capi.SYMBOLS))
    for ret, name, _ in hhg.capi.PROTOTYPES:
        fn = getattr(lib, name)
        assert fn.argtypes is not None, name
        assert (fn.restype is C.c_int) == (ret == "int"), (name, ret, fn.restype)


def _header_structs():
    """{typedef name: [field names in declaration order]} of the structs include/hhg.h defines."""
    with open(HEADER) as h:
        src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", h.read(), flags=re.S)
    return {name: [f for decl in body.split(";") for f in re.findall(r"(\w+)\s*(?:,|$)", decl.strip())]
            for body, name in re.findall(r"typedef\s+struct\s+\w+\s*\{(.*?)\}\s*(\w+)\s*;", src, flags=re.S)}


def _layout(m):
    """(size, [(field, offset, size)]) of a ctypes structure or a numpy record dtype."""
    if isinstance(m, np.dtype):
        return m.itemsize, [(f, m.fields[f][1], m.fields[f][0].itemsize) for f in m.names]
    return C.sizeof(m), [(f, getattr(m, f).offset, getattr(m, f).size) for f, _ in m._fields_]


def test_struct_mirrors_match_compiler_layout(hhg, tmp_path):
    """Every Python mirror of a header struct has the header's fields in order, at the offsets and sizes g++ gives
    them, and the struct's size: a mirror that drifts from the header would hand the library shifted fields."""
    capi = hhg.capi
    mirrors = [("hhg_params", capi.Params), ("hhg_prep_params", capi.PrepParams), ("hhg_msa_params", capi.MsaParams),
               ("hhg_seqdb", capi.SeqDb), ("hhg_admix", capi.Admix), ("hhg_mac_params", capi.MacParams),
               ("hhg_hit", capi.HIT_DTYPE), ("hhg_hit_stats", capi.STATS_DTYPE), ("hhg_topk_rec", capi.TOPK_DTYPE),
               ("hhg_hit", capi.TOPK_DTYPE["hit"]), ("hhg_mac_hit", capi.MAC_HIT_DTYPE),
               ("hhg_stage_stats", capi.STAGE_STATS_DTYPE)]
    fields = _header_structs()
    src = ["#include <cstddef>", "#include <cstdio>", '#include "hhg.h"', "int main() {"]
    for s in sorted({s for s, _ in mirrors}):
        src.append(f'std::printf("{s} %zu\\n", sizeof({s}));')
        src += [f'std::printf("{s} {f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s}*)0)->{f}));' for f in fields[s]]
    (tmp_path / "layout.cpp").write_text("\n".join(src + ["}"]) + "\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", exe,
                           str(tmp_path / "layout.cpp")])
    compiled = {}
    for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines():
        s, *rest = line.split()
        if len(rest) == 1:
            compiled[s] = (int(rest[0]), [])
        else:
            compiled[s][1].append((rest[0], int(rest[1]), int(rest[2])))
    for s, m in mirrors:
        assert _layout(m) == compiled[s], s


def test_sass_is_sm90a_only():
    so = os.path.join(ROOT, "hh-suite_b200", "libhhg.so")
    out = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="GPU present")
def test_no_cpu_fallback(hhg):
    with pytest.raises(hhg.HhgError) as e:
        hhg.Context()
    assert "no CPU fallback" in str(e.value)
