"""CPU: the C-ABI library loads without a GPU and exports exactly the symbols include/mqdet_b200.h declares."""
import os
import re

from util import ROOT


def _declared():
    """name -> parameter count of every declaration, read with a regex of its own (not the loader's parser)."""
    src = open(os.path.join(ROOT, "include", "mqdet_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {name: 0 if params.strip() in ("", "void") else params.count(",") + 1
            for name, params in re.findall(r"\b(mqdet_[a-z0-9_]+)\s*\(([^)]*)\)", src)}


def test_library_loads_and_exports_every_declared_symbol():
    from mqdet_b200 import _lib
    lib = _lib.load()  # binds every name in SIGNATURES; AttributeError if one is missing
    declared = _declared()
    assert declared, "no declarations parsed"
    assert sorted(_lib.SIGNATURES) == sorted(declared), (sorted(set(declared) ^ set(_lib.SIGNATURES)))
    assert {k: len(v[1]) for k, v in _lib.SIGNATURES.items()} == declared
    for name in declared:
        assert hasattr(lib, name)
    assert lib.mqdet_version() >= 100
    assert lib.mqdet_ml_nms_workspace_bytes(5000) > 5000 * 79 * 8


def test_header_types_without_a_binding_raise():
    import ctypes
    import pytest
    from mqdet_b200 import _lib
    sigs = _lib.parse_header("const char* mqdet_a(void);\nvoid mqdet_b(const float* x, int64_t n,\n    int k, void* stream);")
    assert sigs == {"mqdet_a": (ctypes.c_char_p, []),
                    "mqdet_b": (None, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p])}
    with pytest.raises(_lib.MqdetError, match=r"mqdet_c.*double"):
        _lib.parse_header("int mqdet_c(const float* x, double scale, void* stream);")
    with pytest.raises(_lib.MqdetError, match=r"mqdet_d.*size_t"):
        _lib.parse_header("size_t mqdet_d(void);")


def test_gemm_args_struct_matches_header_field_order():
    import ctypes
    from mqdet_b200 import _lib
    src = open(os.path.join(ROOT, "include", "mqdet_b200.h")).read()
    body = src[src.index("typedef struct mqdet_gemm_args {"):src.index("} mqdet_gemm_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    scalar = {"int64_t": ctypes.c_int64, "int32_t": ctypes.c_int32, "float": ctypes.c_float}
    fields = []
    for decl in body.split("{", 1)[1].split(";"):
        decl = decl.strip()
        if not decl:
            continue
        ctype = ctypes.c_void_p if "*" in decl else scalar[decl.split()[0]]
        parts = decl.replace("*", " ").split(",")
        fields.append((parts[0].split()[-1], ctype))
        fields.extend((p.strip(), ctype) for p in parts[1:])
    assert fields == list(_lib.GemmArgs._fields_)


def test_product_path_never_imports_the_oracle():
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "mqdet_b200")):
        for f in files:
            if f.endswith(".py") and re.search(r"^\s*(from|import)\s+oracle\b", open(os.path.join(d, f)).read(), re.M):
                bad.append(f)
    assert not bad, bad


def test_no_cpu_fallback():
    import pytest
    import torch
    from mqdet_b200 import ops
    from mqdet_b200._lib import MqdetError
    with pytest.raises(MqdetError):
        ops.layernorm(torch.zeros(2, 8), torch.ones(8), torch.zeros(8))


def test_entry_points_reject_bad_arguments_without_gpu():
    """Every entry point validates its arguments BEFORE touching CUDA: a bad call returns a negative code and a message in
    mqdet_last_error() (mirrors the reference's AT_ERROR / TORCH_CHECK behaviour), also on a machine without a GPU."""
    import ctypes
    from mqdet_b200 import _lib
    lib = _lib.load()
    nul = ctypes.c_void_p(0)
    one = ctypes.c_void_p(16)  # never dereferenced: the checks fail first

    def expect(rc, needle):
        assert rc < 0
        msg = lib.mqdet_last_error().decode()
        assert needle in msg, msg

    g = _lib.GemmArgs()
    expect(lib.mqdet_gemm_f16(ctypes.byref(g), 0, nul), "null pointer")
    g.A = g.B = g.C = 16
    g.M, g.N, g.K = 4, 4, 0
    expect(lib.mqdet_gemm_f16(ctypes.byref(g), 0, nul), "empty problem")
    g.K, g.lda, g.ldb, g.ldc, g.nb1, g.nb2 = 12, 12, 12, 4, 1, 1   # K % 8 != 0
    expect(lib.mqdet_gemm_f16(ctypes.byref(g), 0, nul), "multiples of 8")
    g.K = g.lda = g.ldb = 16
    expect(lib.mqdet_gemm_f16(ctypes.byref(g), 7, nul), "unknown impl")
    expect(lib.mqdet_layernorm(nul, 0, 8, nul, nul, 1e-5, 1, 8, nul, nul, 8, 0, nul), "null pointer")
    expect(lib.mqdet_softmax_rows(one, _lib.F16, 8, one, 8, 1, 8, 8, 1.0, nul, 0, 0.0, 0.0, nul), "fp32")   # fp16 scores
    expect(lib.mqdet_swin_window_attn(one, one, one, 1, 14, 14, 3, 8, 0, 1.0, one, nul), "window 7 (Swin-T) or 12 (Swin-L)")
    expect(lib.mqdet_biattn_image(one, 8, 8, one, 8, 8, 8, nul, 0, one, 8, 8, 8, nul, nul, nul, 0, 0, nul, 0.0, one, 8, 8, one,
                                  one, 1, 8, 100, 100, nul), "T % 8 == 0")
    expect(lib.mqdet_biattn_text_vn(one, 8, 8, 8, one, 8, 8, 8, one, 8, 0, 8, nul, nul, 0, 0.0, one, 8, 8, 8, 1, 1, 256, 100, nul),
           "null pointer")
    expect(lib.mqdet_gather_detections(one, one, one, one, one, 1, 256, 128, 64, one, nul), "det_rows")
    expect(lib.mqdet_dcn_cols(one, nul, 0, one, 5, 1, 128, 1, one, nul), "C must be 256")
    expect(lib.mqdet_dcn_conv(one, nul, 0, one, 5, 1, 128, 1, one, one, one, one, nul), "C must be 256")
    expect(lib.mqdet_dcn_conv(one, nul, 0, one, 5, 1, 256, 4, one, one, one, one, nul), "1..3 jobs")
    expect(lib.mqdet_conv3x3_small(one, one, one, one, 5, 1, 256, 40, one, 64, nul), "O <= 32")
    expect(lib.mqdet_contrastive_mask(one, one, 1, 1, 300, 256, nul), "bad args")                # Tmax < T
