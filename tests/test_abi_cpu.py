"""CPU: the C-ABI shared library loads without a GPU and exports every symbol include/otter_b200.h declares;
argument validation returns error codes (never throws / exits); no compute is launched here."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "otter_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(otb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from otter_b200 import _lib
    lib = _lib.load()
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/otter_b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == syms, "ctypes SIGNATURES table out of sync with the header"
    assert lib.otb_compiled_arch() == 90 and lib.otb_version() >= 1


def test_struct_layouts_match_header():
    from otter_b200 import _lib
    lib = _lib.load()
    # the C compiler's layout (otb_abi_sizeof) vs the ctypes mirror, and vs the header's field lists
    assert lib.otb_abi_sizeof(0) == C.sizeof(_lib.GemmEpilogue) == 6 * 8 + 4 * 8 + 6 * 4
    assert lib.otb_abi_sizeof(1) == C.sizeof(_lib.AttnDesc) == 6 * 8 + 4 * 8 + 17 * 4 + 4 + 2 * 4
    assert lib.otb_abi_sizeof(2) == C.sizeof(_lib.AttnGrads) == 5 * 8 + 4 * 8 + 8 * 4


def test_invalid_arguments_return_error_codes():
    from otter_b200 import _lib
    lib = _lib.load()
    e = _lib.GemmEpilogue()
    rc = lib.otb_gemm_bf16(None, 0, 0, None, 0, 0, 0, 0, 0, C.byref(e), None)
    assert rc == 1 and b"otb_gemm_bf16" in lib.otb_last_error()
    # valid shapes, 16-byte aligned A / B, an output 2 bytes past a 16-byte boundary: rejected before any launch
    e.out, e.ld_out = 0x10002, 128
    rc = lib.otb_gemm_bf16(0x10000, 0, 128, 0x20000, 0, 128, 128, 128, 128, C.byref(e), None)
    assert rc == 1 and b"aligned" in lib.otb_last_error()
    # bias / residual / aux_in / aux_out are read or written in 16 B vectors by the epilogue.  M = 0: the alignment
    # check must come before the shape check, or the message below names the shape instead of the pointer.
    launches = lib.otb_launch_count()
    for name in ("bias", "residual", "aux_in", "aux_out"):
        e = _lib.GemmEpilogue()
        e.out, e.ld_out = 0x10000, 128
        e.ld_aux_in = e.ld_aux_out = e.ld_res = 128
        setattr(e, name, 0x30000 + 4)
        rc = lib.otb_gemm_bf16(0x10000, 0, 128, 0x20000, 0, 128, 0, 128, 128, C.byref(e), None)
        msg = lib.otb_last_error()
        assert rc == 1 and name.encode() in msg and b"aligned" in msg, (name, msg)
    assert lib.otb_launch_count() == launches
    assert lib.otb_text_time(None, 0, 0, 1, None, None) == 1
    assert lib.otb_layernorm_fwd(None, 0, None, None, None, 0, None, None, 0, 0, 1e-5, None) == 1
    d = _lib.AttnDesc()
    assert lib.otb_attn_fwd(C.byref(d), None) == 1
    assert lib.otb_ln_chunks(2048, 4096) >= 1 and lib.otb_dot_blocks() > 0
    assert lib.otb_launch_count() == 0      # nothing was launched by the calls above


def test_ops_reject_cpu_tensors_loudly():
    import torch
    from otter_b200 import _lib
    from otter_b200 import functional as F
    with pytest.raises(_lib.OtbError, match="CUDA tensor"):
        F.linear_fwd(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))


def test_sass_is_hopper_native():
    """The built library must contain sm_90a warpgroup tensor-core / TMA / mbarrier machine code (wgmma ->
    HGMMA, TMA -> UTMALDG / UTMASTG, mbarrier -> SYNCS) and no legacy mma.sync path (HMMA)."""
    import shutil
    import subprocess
    from otter_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA.64x128x16.F32.BF16", "HGMMA.64x64x16.F32.BF16", "UTMALDG", "UTMASTG", "SYNCS"):
        assert mnemonic in sass, f"{mnemonic} missing from the SASS"
    assert "HMMA." not in sass, "legacy mma.sync (HMMA) found"


def test_integration_guide_names_every_entry_point():
    """INTEGRATION.md's table (entry point -> reference file:line it replaces) covers the whole header."""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "otter_b200.h")).read()
    doc = open(os.path.join(root, "INTEGRATION.md")).read()
    syms = sorted(set(re.findall(r"\b(otb_[a-z0-9_]+)\s*\(", hdr)))
    assert len(syms) >= 50
    assert [s for s in syms if s not in doc] == []
