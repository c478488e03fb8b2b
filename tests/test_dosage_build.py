"""CPU checks of what the compiler made of the dosage path and of how the R shim reaches it: the byte-operand kernels of
bsg_dosage.cu compile for sm_90a without spills, k_dmv / k_dmvT are IMMA.16832.U8.S8 code, the identity-selection k_dmvT
loads through the tensor memory accelerator (UTMALDG) and the column-list k_dmvT through bulk copies (UBLKCP); the shim
registers _bigsnpr_prod_and_rowSumsSq2 with the reference's arity and lets _bigsnpr_bed_randomSVD_gpu take an FBM."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bigsnpr_b200", "csrc")


@pytest.fixture(scope="module")
def built():
    from bigsnpr_b200 import build

    return build.build()


def _sass_by_function(so):
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", out)
    return {parts[i]: parts[i + 1] for i in range(1, len(parts) - 1, 2)}


def test_dosage_kernels_sass(built):
    fn = _sass_by_function(built)
    dmv = [b for name, b in fn.items() if "3dos5k_dmvE" in name]
    tma = [b for name, b in fn.items() if "3dos6k_dmvTILb0E" in name]
    lst = [b for name, b in fn.items() if "3dos6k_dmvTILb1E" in name]
    assert len(dmv) == 1 and len(tma) == 1 and len(lst) == 1, sorted(n for n in fn if "dos" in n)
    for body in dmv + tma + lst:
        assert "IMMA.16832.U8.S8" in body
    assert "UTMALDG" in tma[0]
    assert "UBLKCP" in lst[0] and "UTMALDG" not in lst[0]


def test_dosage_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        "-I", os.path.join(ROOT, "include"), "-I", CSRC, os.path.join(CSRC, "bsg_dosage.cu"),
                        "-o", str(tmp_path / "bsg_dosage.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    props = re.findall(r"Function properties for (\S+)\n[^\n]*?(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    names = [p[0] for p in props]
    for k in ("k_dmvE", "k_dmvTILb0E", "k_dmvTILb1E", "k_digits_rows", "k_proj_literal"):
        assert any(k in nm for nm in names), (k, names)
    for nm, st, ld in props:
        assert st == "0" and ld == "0", nm


def test_shim_projection_and_fbm_randomsvd_entry_points(tmp_path):
    import ctypes

    from tests.test_abi import build_shim_with_minir

    so = build_shim_with_minir(tmp_path)
    L = ctypes.CDLL(so)
    L.R_init_bigsnpr_hotpath(None)
    L.minir_routine_name.restype = ctypes.c_char_p
    table = {L.minir_routine_name(i).decode(): L.minir_routine_nargs(i) for i in range(L.minir_routine_count())}
    assert table["_bigsnpr_prod_and_rowSumsSq2"] == 6
    assert len([nm for nm in table if nm.endswith("_gpu")]) == 6
    src = open(os.path.join(ROOT, "r_shim", "bigsnpr_shim.c")).read()

    def body(fn):
        b = src[src.index("SEXP %s(" % fn):]
        return b[:b.index("\n}\n")]

    assert "fbm_handle_of(BM)" in body("_bigsnpr_prod_and_rowSumsSq2")
    assert "bsg_prod_and_rowsumssq2(" in body("_bigsnpr_prod_and_rowSumsSq2")
    assert "any_handle(obj_bed)" in body("_bigsnpr_bed_randomSVD_gpu")
