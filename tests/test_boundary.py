"""CPU: the drop-in boundary.  The C-ABI library loads, exports every symbol
include/fi_epp.h declares, fails loudly without a CUDA device (no CPU fallback), and
the product never touches oracle/."""
import ctypes as C
import os
import re

import pytest

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import default_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "fi_epp.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fi_epp_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = abi.load()
    declared = _declared_symbols()
    assert len(declared) >= 20
    bound = {name for name, _, _ in abi.SYMBOLS}
    assert set(declared) == bound, set(declared) ^ bound
    for name in declared:
        assert getattr(lib, name) is not None


def test_struct_layouts_match_header_sizes():
    # sizes implied by include/fi_epp.h (natural alignment, little-endian x86-64)
    assert C.sizeof(abi.fi_pick) == 16
    assert C.sizeof(abi.fi_index_op) == 16
    assert C.sizeof(abi.fi_endpoint_state) == 24
    assert C.sizeof(abi.fi_scorer) == 8
    assert C.sizeof(abi.fi_profile) == 32 + 8 + 8 * abi.FI_EPP_MAX_SCORERS + 4 * abi.FI_EPP_MAX_FILTERS
    assert C.sizeof(abi.fi_label_bit) == 128
    cfg = default_config()
    assert cfg.struct_size == C.sizeof(abi.fi_epp_config)  # the library's own sizeof


def test_abi_version_and_status_strings():
    lib = abi.load()
    assert lib.fi_epp_abi_version() == abi.FI_EPP_ABI_VERSION
    assert b"no CPU fallback" in lib.fi_epp_status_string(abi.FI_ERR_CUDA)


def test_create_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    cfg = default_config()
    h = C.c_void_p()
    rc = abi.load().fi_epp_create(C.byref(cfg), C.byref(h))
    assert rc == abi.FI_ERR_CUDA and not h.value


def test_create_rejects_bad_configs_before_touching_the_device():
    lib = abi.load()
    for mutate in (lambda c: setattr(c, "struct_size", 8), lambda c: setattr(c, "max_blocks", 5000),
                   lambda c: setattr(c, "endpoint_count", 0), lambda c: setattr(c, "n_profiles", 9)):
        cfg = default_config()
        mutate(cfg)
        h = C.c_void_p()
        assert lib.fi_epp_create(C.byref(cfg), C.byref(h)) == abi.FI_ERR_INVALID


def test_product_never_references_the_oracle():
    pkg = os.path.join(ROOT, "fusioninfer_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                for ln in text.splitlines():
                    code = ln.split("//")[0].split("#")[0] if not ln.lstrip().startswith(("//", "#", "*", '"')) else ""
                    assert "epp_oracle" not in code and "oracle/" not in code, (f, ln)
    mk = open(os.path.join(ROOT, "Makefile")).read()
    # the link rule of libfi_epp.so: its prerequisites and recipe must not mention oracle/
    rule = mk[mk.index("$(LIB): "):]
    rule = rule[: rule.index("\n\n")]
    assert "oracle" not in rule, rule


def test_kernels_are_built_for_sm_90a():
    so = abi.LIB_PATH
    import shutil
    import subprocess

    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    out = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_header_is_c_and_links_from_a_c_program(tmp_path):
    """include/fi_epp.h compiles as strict C99 and a plain C program links libfi_epp.so and drives the
    configuration entry points (tests/c/abi_check.c) — the binding a cgo file would make, without Go."""
    import shutil
    import subprocess

    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "fusioninfer_b200", "lib")
    exe = str(tmp_path / "abi_check")
    cmd = [gcc, "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(root, "include"),
           os.path.join(root, "tests", "c", "abi_check.c"), "-L", libdir, "-lfi_epp", f"-Wl,-rpath,{libdir}",
           "-Wl,--allow-shlib-undefined", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    env = dict(os.environ)
    cuda_lib = "/usr/local/cuda/lib64"
    env["LD_LIBRARY_PATH"] = cuda_lib + ":" + env.get("LD_LIBRARY_PATH", "")
    r = subprocess.run([exe], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi_check:" in r.stdout
