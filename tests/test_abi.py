"""The C-ABI library builds for sm_90a, loads, exports every symbol of include/vcalloc.h, and — on a box
without a GPU — refuses to compute instead of falling back to a CPU path."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from volcano_b200.build import build_lib
    from volcano_b200 import engine
    build_lib()
    return engine.load_library()


def test_exports_every_declared_symbol(lib):
    from volcano_b200 import abi
    hdr = open(os.path.join(ROOT, "include", "vcalloc.h")).read()
    declared = set(re.findall(r"\b(vc_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"vc_plugin_option", "vc_tasks"}  # "vc_tasks (best-effort, gated)" is prose in a comment
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(lib, name), f"libvcalloc.so lacks {name}"
    assert declared == set(abi.SYMBOLS), declared ^ set(abi.SYMBOLS)
    assert lib.vc_abi_version() == abi.VC_ABI_VERSION


def test_struct_sizes_match_header(lib):
    from volcano_b200 import abi
    assert C.sizeof(abi.vc_decision) == 24 and C.sizeof(abi.vc_visit) == 16
    assert C.sizeof(abi.vc_dims) == 12 * 4
    assert C.sizeof(abi.vc_conf) == 4 + 16 * 12 + 4 + 16 * 4 + 5 * 4 + 4 * 4 + 4 + 5 * 4 + 4 + (4 + 16 * 4 + 4) + 8  # 408
    assert C.sizeof(abi.vc_hypernodes) == 16 + 7 * 8


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volcano_b200 import abi, engine
    from volcano_b200.synth import make_snapshot
    assert lib.vc_init(0) == abi.VC_ENODEV
    assert b"no CPU path" in lib.vc_last_error()
    with pytest.raises(engine.VcError) as ei:
        engine.gpu_engine(make_snapshot("tiny"))
    assert ei.value.code == abi.VC_ENODEV


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "volcano_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert "pyoracle" not in src and "oracle/" not in src and "import oracle" not in src, f


def test_graft_entry_build_is_consistent():
    """build() is what the driver runs on CPU every round: it must agree with the header's ABI version."""
    import __graft_entry__ as g
    g.build()


def _header_structs():
    """typedef struct vc_x { ... } vc_x; -> {name: [field, ...]} parsed from include/vcalloc.h (comments stripped)."""
    hdr = open(os.path.join(ROOT, "include", "vcalloc.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    out = {}
    for m in re.finditer(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*(\w+)\s*;", hdr, flags=re.S):
        name, body = m.group(3), m.group(2)
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            # "const double *a, *b" / "int32_t x[16]" / "vc_plugin_option plugins[VC_MAX_PLUGINS]"
            decl = re.sub(r"^(const\s+)?(struct\s+)?\w+\s+", "", decl, count=1)
            for d in decl.split(","):
                d = d.strip().lstrip("*").strip()
                d = re.sub(r"^const\s+", "", d)
                d = re.sub(r"\[.*\]$", "", d).strip().lstrip("*").strip()
                if d:
                    fields.append(d)
        out[name] = fields
    return out


def test_ctypes_mirror_matches_the_header_field_by_field(tmp_path):
    """Every struct of include/vcalloc.h: size and the offset of every field as gcc lays them out vs the ctypes mirror in
    volcano_b200/abi.py (the layouts are written twice by hand; this is the check that they agree)."""
    import shutil
    import subprocess
    from volcano_b200 import abi
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    structs = _header_structs()
    assert {"vc_dims", "vc_nodes", "vc_tasks", "vc_jobs", "vc_queues", "vc_classes", "vc_conf", "vc_decision", "vc_visit",
            "vc_stats", "vc_hypernodes", "vc_running_tasks"} <= set(structs), sorted(structs)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "vcalloc.h"', "int main(void) {"]
    for name, fields in structs.items():
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        for f in fields:
            lines.append(f'  printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(ln.split() for ln in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    checked = 0
    for name, fields in structs.items():
        mirror = getattr(abi, name, None)
        assert mirror is not None, f"abi.py lacks {name}"
        assert C.sizeof(mirror) == int(got[name]), (name, C.sizeof(mirror), got[name])
        assert [f for f, _ in mirror._fields_] == fields, (name, [f for f, _ in mirror._fields_], fields)
        for f in fields:
            assert getattr(mirror, f).offset == int(got[f"{name}.{f}"]), (name, f)
            checked += 1
    assert checked >= 140
