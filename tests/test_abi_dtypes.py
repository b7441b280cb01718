"""CPU test of the C ABI's dtype dispatch: every entry point that takes a dtype code refuses a code it has no kernel for, before any
CUDA call, with a non-zero return and "<op>: unsupported dtype <code>" (include/romab200.h).  The calls run in a subprocess that sees no
CUDA device, so a code that slipped through could not reach a GPU either: it would fail later, with a different message."""
import json
import os
import subprocess
import sys

import pytest

from roma_b200 import cabi
from roma_b200.cabi import RB_F16, RB_F16S, RB_F32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD = 7            # outside the enum
ADDR = 1 << 20     # stands in for a device pointer where an entry point refuses NULL; never dereferenced

# (entry point, struct, fields that pass the entry point's shape checks, dtype field, refused codes)
CASES = [
    ("gemm", "rb_gemm_args", dict(A=ADDR, B=ADDR, C=ADDR, M=16, N=16, K=16, lda=16, ldb=16, ldc=16, dtype_ab=RB_F32), "dtype_c", [BAD, -1]),
    ("gemm", "rb_gemm_args", dict(A=ADDR, B=ADDR, C=ADDR, M=16, N=16, K=16, lda=16, ldb=16, ldc=16, dtype_ab=RB_F16), "dtype_c", [BAD]),
    ("gemm", "rb_gemm_args", dict(A=ADDR, B=ADDR, C=ADDR, R=ADDR, M=16, N=16, K=16, lda=16, ldb=16, ldc=16, ldr=16, dtype_ab=RB_F32,
                                  dtype_c=RB_F32), "dtype_r", [RB_F16S, BAD]),
    ("layernorm", "rb_layernorm_args", dict(rows=4, cols=8, ldx=8, ldy=8, dtype_x=RB_F32), "dtype_y", [BAD]),
    ("layernorm", "rb_layernorm_args", dict(rows=4, cols=8, ldx=8, ldy=8, dtype_y=RB_F32), "dtype_x", [RB_F16, RB_F16S, BAD]),
    ("softmax_rows", "rb_softmax_args", dict(rows=4, cols=8, lds=8), "dtype", [RB_F16S, BAD]),
    ("flash_attn", "rb_flash_attn_args", dict(ld_qkv=192, ld_out=64, batch=1, n_tokens=64, heads=1, head_dim=64), "dtype", [RB_F32, BAD]),
    ("row_norms", "rb_rownorm_args", dict(rows=4, cols=8, ldx=8), "dtype", [RB_F16S, BAD]),
    ("copy2d", "rb_copy2d_args", dict(rows=4, cols=8, lds=8, ldd=8, dtype_dst=RB_F32), "dtype_src", [RB_F16S, BAD]),
    ("copy2d", "rb_copy2d_args", dict(rows=4, cols=8, lds=8, ldd=8, dtype_src=RB_F32), "dtype_dst", [RB_F16S, BAD]),
    ("conv3x3_first", "rb_conv_first_args", dict(batch=1, height=8, width=8, cout=64), "dtype_out", [BAD]),
    ("maxpool2x2_padded", "rb_maxpool_args", dict(batch=1, height=4, width=4, channels=8), "dtype", [BAD]),
    ("im2col_patch", "rb_im2col_args", dict(batch=1, height=14, width=14, patch=14, ldo=588), "dtype_out", [RB_F16S, BAD]),
    ("cls_to_flow_refine", "rb_cls_args", dict(rows=4, ldl=5, res=2), "dtype", [RB_F16S, BAD]),
    ("refiner_prologue", "rb_refiner_prologue_args", dict(ldf=8, n_img=2, ldd=16, D=1, h=4, w=4, cf=8, emb=0, radius=0), "dtype", [RB_F16S, BAD]),
    ("local_corr", "rb_local_corr_args", dict(ldf0=8, ldf1=8, ldo=25, batch=1, h=4, w=4, c=8, radius=2, dtype_out=RB_F32), "dtype_f", [RB_F16S, BAD]),
    ("dwconv5x5_relu", "rb_dwconv_args", dict(ldi=8, ldo=8, ldw=8, batch=1, h=8, w=8, c=8), "dtype", [RB_F16S, BAD]),
    ("refiner_block_small", "rb_refiner_block_small_args", dict(ld=24, ldw=24, batch=1, h=8, w=8, c=24), "dtype", [RB_F16S, BAD]),
    ("refiner_block_c144", "rb_refiner_block_c144_args", dict(ld=144, ldw=144, ld_pw=144, batch=1, h=8, w=8, c=144), "dtype",
     [RB_F32, RB_F16S, BAD]),
    ("refiner_tail", "rb_refiner_tail_args", dict(ldd=8, ldw=8, rows=4, c=8), "dtype", [RB_F16S, BAD]),
    ("transpose", "rb_transpose_args", dict(rows=32, cols=32, lds=32, ldd=32, batch0=1, batch1=1), "dtype", [RB_F16S, BAD]),
]

_CHILD = r"""
import ctypes, json, sys
from roma_b200 import cabi
lib = cabi.load_library()
out = []
for fn, struct, fields, code_field, code in json.load(sys.stdin):
    args = cabi.STRUCTS[struct]()
    for k, v in fields.items():
        setattr(args, k, v)
    setattr(args, code_field, code)
    rc = getattr(lib, "romab200_" + fn)(ctypes.byref(args), None)
    out.append([rc, lib.romab200_last_error().decode()])
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def results():
    calls = [(fn, struct, fields, code_field, code) for fn, struct, fields, code_field, codes in CASES for code in codes]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable, *flags, "-c", _CHILD], input=json.dumps(calls), capture_output=True, text=True, cwd=ROOT, env=env,
                         timeout=600)
    assert res.returncode == 0, res.stderr
    return dict(zip([(c[0], c[3], c[4]) for c in calls], json.loads(res.stdout.strip().splitlines()[-1])))


@pytest.mark.parametrize("fn, field, code", [(fn, field, code) for fn, _, _, field, codes in CASES for code in codes])
def test_unsupported_dtype_is_refused(results, fn, field, code):
    rc, msg = results[(fn, field, code)]
    assert rc != 0 and msg == f"{fn}: unsupported dtype {code}", (rc, msg)


def test_every_struct_with_a_dtype_code_is_covered():
    with_code = {s for s, fs in cabi.STRUCT_FIELDS.items() if any(f == "dtype" or f.startswith("dtype_") for f, _ in fs)}
    assert with_code == {struct for _, struct, _, _, _ in CASES}
