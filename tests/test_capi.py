"""The C-ABI library loads and exports every symbol include/controllora_b200.h declares; the ctypes mirrors of the
argument structs have the C layout.  No compute calls (no GPU here)."""
import ctypes
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "controllora_b200.h"


def declared_functions():
    text = HEADER.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = re.findall(r"^\s*(?:const\s+char\*|int64_t|int)\s+(cl_[a-z0-9_]+)\s*\(", text, flags=re.M)
    assert len(names) >= 40, names
    return sorted(set(names))


def test_all_declared_symbols_are_exported(built_lib):
    lib = ctypes.CDLL(str(built_lib))
    missing = [n for n in declared_functions() if not hasattr(lib, n)]
    assert not missing, f"declared in the header but not exported: {missing}"


def test_abi_version_and_error_string(built_lib):
    """ABI 101: the GroupNorm entry points take no scratch argument and cl_groupnorm_ws_bytes is gone."""
    from controllora_b200 import _lib

    lib = _lib.lib()
    assert lib.cl_version() == 101
    assert isinstance(lib.cl_last_error(), bytes)
    assert _lib.launch_count() >= 0


def test_struct_layouts_match_c(built_lib, tmp_path):
    from controllora_b200 import _lib

    src = tmp_path / "sz.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "controllora_b200.h"\n'
        "int main(){printf(\"%zu %zu %zu %zu %zu %zu %zu\\n\", sizeof(cl_gemm_args), sizeof(cl_attn_fwd_args), sizeof(cl_attn_bwd_args),"
        " sizeof(cl_pack_desc), offsetof(cl_gemm_args, out), offsetof(cl_attn_bwd_args, scale), offsetof(cl_pack_desc, row_off));return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = [ctypes.sizeof(_lib.GemmArgs), ctypes.sizeof(_lib.AttnFwdArgs), ctypes.sizeof(_lib.AttnBwdArgs),
            ctypes.sizeof(_lib.PackDesc), _lib.GemmArgs.out.offset, _lib.AttnBwdArgs.scale.offset, _lib.PackDesc.row_off.offset]
    assert got == want


def test_invalid_arguments_are_rejected_without_a_gpu(built_lib):
    """Argument validation happens before any CUDA call: status < 0 and a message, never a crash."""
    from controllora_b200 import _lib

    lib = _lib.lib()
    args = _lib.GemmArgs()
    assert lib.cl_gemm(ctypes.byref(args), None) == -1
    assert b"null" in lib.cl_last_error()
    a = _lib.AttnFwdArgs()
    assert lib.cl_attn_fwd(ctypes.byref(a), None) == -1


def test_ops_fail_loudly_without_cuda():
    """There is no CPU fallback: CPU tensors are refused."""
    import pytest
    import torch

    from controllora_b200 import _lib, ops

    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    with pytest.raises(_lib.CLError):
        ops.gemm(torch.zeros(128, 64, dtype=torch.bfloat16), torch.zeros(64, 64, dtype=torch.bfloat16))


def test_every_entry_point_is_listed_in_the_integration_table():
    """INTEGRATION.md's C-ABI table (entry point -> reference call site it replaces) stays in step with the header."""
    doc = (ROOT / "INTEGRATION.md").read_text()
    words = set(re.findall(r"cl_[a-z0-9_]+", doc))
    expanded = set(words)
    for w in words:                                   # `cl_attn_fwd`, `cl_groupnorm_fwd/bwd`, `cl_conv_out(_bwd)`, `cl_upsample2x_*`
        for m in re.finditer(re.escape(w) + r"/([a-z0-9_]+)", doc):
            expanded.add(w.rsplit("_", 1)[0] + "_" + m.group(1))
        for m in re.finditer(re.escape(w) + r"\((_[a-z0-9_]+)\)", doc):
            expanded.add(w + m.group(1))
    utility = {"cl_last_error", "cl_version", "cl_launch_count", "cl_gemm_split_hint", "cl_bf16_to_f32", "cl_f32_to_bf16", "cl_nchw_to_nhwc",
               "cl_nhwc_to_nchw_f32"}                  # housekeeping + the "layout casts" of the elementwise row
    missing = [n for n in declared_functions() if n not in expanded and n not in utility and not any(n.startswith(w[:-1]) for w in words if w.endswith("_"))]
    assert not missing, f"declared in the header but absent from INTEGRATION.md's table: {missing}"
