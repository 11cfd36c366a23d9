"""The C-ABI shared library loads without a GPU and exports every symbol that
include/sutro_b200.h declares (no compute calls here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "sutro_b200.h")
LIB = os.path.join(ROOT, "sutro_b200", "libsutro_b200.so")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = set(re.findall(r"\b(sb200_[a-z0-9_]+)\s*\(", text))
    names -= {"sb200_progress_fn"}
    return sorted(names)


def test_header_declares_the_expected_surface():
    names = declared_symbols()
    for must in ["sb200_engine_create", "sb200_engine_run", "sb200_tokenizer_encode",
                 "sb200_tokenizer_decode", "sb200_gemm_bf16_tn", "sb200_attn_decode",
                 "sb200_attn_prefill", "sb200_rope_kv_write", "sb200_rmsnorm",
                 "sb200_fsm_build_mask", "sb200_last_error"]:
        assert must in names


@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built (run __graft_entry__.build())")
def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(LIB)
    missing = [n for n in declared_symbols() if not hasattr(lib, n)]
    assert not missing, missing
    lib.sb200_abi_version.restype = ctypes.c_int
    assert lib.sb200_abi_version() == 1
    lib.sb200_last_error.restype = ctypes.c_char_p
    assert lib.sb200_last_error() is not None


@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built")
def test_python_binding_table_matches_header():
    from sutro_b200 import _lib, engine  # noqa: F401  (engine registers its entry points)
    assert set(_lib.exported_symbols()) == set(declared_symbols())
    _lib.lib()


@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built")
@pytest.mark.parametrize("hq,hkv,msg", [
    (12, 4, "unsupported GQA group size 3"),
    (12, 0, "hq=12 not a multiple of hkv=0"),
])
def test_attention_launchers_reject_unsupported_gqa_groups(hq, hkv, msg):
    """The GQA group is checked before any CUDA call, so this needs no GPU."""
    lib = ctypes.CDLL(LIB)
    lib.sb200_last_error.restype = ctypes.c_char_p
    ints = (ctypes.c_int32 * 4)()
    scale = ctypes.c_float(1.0)
    calls = {
        "attn_decode": lambda: lib.sb200_attn_decode(
            None, None, None, ints, 1, ints, ints, 1, hq, hkv, scale, None),
        "attn_prefill": lambda: lib.sb200_attn_prefill(
            None, None, None, ints, 1, ints, 1, ints, ints, ints, ints, hq, hkv, scale, None),
        "attn_prefill_dense": lambda: lib.sb200_attn_prefill_dense(
            None, 1, None, None, 0, 1, 0, ints, 1, ints, ints, ints, hq, hkv, scale, None),
    }
    for who, call in calls.items():
        assert call() == -1, who
        assert lib.sb200_last_error().decode() == f"{who}: {msg}"


@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built")
def test_attn_prefill_stub_names_the_dense_kernel():
    """sb200_attn_prefill stays in ABI version 1 without a kernel behind it: with a supported GQA
    group it fails before any CUDA call, so this needs no GPU."""
    lib = ctypes.CDLL(LIB)
    lib.sb200_last_error.restype = ctypes.c_char_p
    ints = (ctypes.c_int32 * 4)()
    assert lib.sb200_attn_prefill(None, None, None, ints, 1, ints, 1, ints, ints, ints, ints, 32,
                                  8, ctypes.c_float(1.0), None) == -1
    assert lib.sb200_last_error().decode() == (
        "sb200_attn_prefill: the library has no paged prefill attention; use "
        "sb200_attn_prefill_dense")


@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built")
def test_decode_force_variant_is_still_exported():
    """sb200_attn_decode_force_variant stays in ABI version 1 as a no-op (one decode kernel)."""
    lib = ctypes.CDLL(LIB)
    fn = lib.sb200_attn_decode_force_variant
    fn.restype = None
    fn.argtypes = [ctypes.c_int]
    for v in (0, 1, 2):
        fn(v)


def test_no_product_module_imports_the_oracle():
    pkg = os.path.join(ROOT, "sutro_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def test_ctypes_struct_layouts_match_the_header(tmp_path):
    """The Python mirrors of the C structs (engine.py) against the header itself: a probe
    compiled with gcc prints sizeof/offsetof for every field."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    from sutro_b200 import engine as E
    mirrors = {"sb200_engine_config": E.EngineConfigC, "sb200_engine_weights": E.EngineWeightsC,
               "sb200_job": E.JobC, "sb200_job_stats": E.JobStatsC, "sb200_result": E.ResultC,
               "sb200_sample_args": E.SampleArgsC}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void){"]
    for cname, mirror in mirrors.items():
        lines.append(f'printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, *_ in mirror._fields_:
            lines.append(f'printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines.append("return 0;}")
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    seen = 0
    for line in out.splitlines():
        cname, what, value = line.split()
        mirror = mirrors[cname]
        want = ctypes.sizeof(mirror) if what == "size" else getattr(mirror, what).offset
        assert int(value) == want, (cname, what, value, want)
        seen += 1
    assert seen == sum(len(m._fields_) + 1 for m in mirrors.values())
