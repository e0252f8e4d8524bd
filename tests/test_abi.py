"""The C-ABI library loads without a GPU and exports every symbol include/sgformer_b200.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "sgformer_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sgf_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_expected_surface():
    syms = declared_symbols()
    for s in ("sgf_csr_build", "sgf_spmm", "sgf_gemm_nt", "sgf_gemm_tn", "sgf_ln_fwd", "sgf_bn_fwd", "sgf_subgraph"):
        assert s in syms


def test_library_builds_loads_and_exports_everything():
    import __graft_entry__ as g
    g.build()
    from sgformer_b200 import _lib
    lib = ctypes.CDLL(_lib.lib_path())
    for s in declared_symbols():
        assert hasattr(lib, s), f"libsgformer_b200.so does not export {s}"
    assert set(declared_symbols()) == set(_lib._SIGS), "ctypes signature table and header disagree"
    lib.sgf_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.sgf_version()


def test_struct_layouts_match_the_header():
    """sizeof(sgf_gemm_nt_args / sgf_gemm_tn_args) as compiled by gcc == the ctypes mirrors."""
    import subprocess
    import tempfile
    from sgformer_b200 import _lib
    src = '#include <stdio.h>\n#include "sgformer_b200.h"\nint main(){printf("%zu %zu\\n", sizeof(sgf_gemm_nt_args), sizeof(sgf_gemm_tn_args));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "s")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        a, b = map(int, subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split())
    assert a == ctypes.sizeof(_lib.GemmNtArgs) and b == ctypes.sizeof(_lib.GemmTnArgs)


def test_no_cpu_fallback():
    """Product modules refuse CPU execution when no GPU exists instead of silently computing elsewhere."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from sgformer_b200 import large as L
    from sgformer_b200.medium import full_attention_conv
    m = L.SGFormer(8, 16, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.randn(4, 8), torch.zeros(2, 3, dtype=torch.long))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        full_attention_conv(torch.randn(4, 1, 8), torch.randn(4, 1, 8), torch.randn(4, 1, 8))


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "sgformer_b200")):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", text, flags=re.M), f"{f} imports oracle/"
                assert "kernel_emu" not in text, f"{f} references the test-only kernel emulation"


def test_wrappers_around_the_model_fail_loudly_without_cuda():
    """K10 / K11 wrappers (pyg_utils, eval, kernels.eval_acc) have no CPU path: CPU tensors raise instead of falling back."""
    import pytest
    import torch

    from sgformer_b200 import kernels as K
    from sgformer_b200 import pyg_utils as U

    ei = torch.tensor([[0, 1, 2], [1, 1, 0]])
    for call in (lambda: U.to_undirected(ei, num_nodes=3), lambda: U.remove_self_loops(ei), lambda: U.add_self_loops(ei, num_nodes=3),
                 lambda: U.subgraph(torch.tensor([0, 1]), ei, relabel_nodes=True, num_nodes=3),
                 lambda: K.eval_acc(torch.zeros(3, 2), torch.zeros(3, 1, dtype=torch.long))):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()
    with pytest.raises(NotImplementedError):
        U.remove_self_loops(ei, torch.zeros(3))
