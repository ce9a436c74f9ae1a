"""C-ABI surface (no GPU needed): the library loads and exports every symbol include/vdb200.h declares,
and the ctypes signature table covers exactly that set."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "vdb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(vdb_[a-z0-9_]+)\s*\(", src))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    from vdb200 import _lib
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(_lib.lib, s), f"{s} declared in include/vdb200.h but not exported by libvdb200.so"
    assert set(_lib.SIGNATURES) == syms, sorted(set(_lib.SIGNATURES) ^ syms)
    assert _lib.lib.vdb_version().startswith(b"vdb200")


def test_host_side_argument_checks_without_gpu():
    """Entry points validate arguments before touching the device: bad calls return VDB_ERR_INVALID + a message."""
    from vdb200._lib import lib
    assert lib.vdb_ddim_cfg_step(None, None, None, None, None, None, 1.0, 1.0, None, None, None, 0, None) == 1
    assert b"ddim_cfg_step" in lib.vdb_last_error()
    assert lib.vdb_gemm_bf16(None, 0, 0, 0, None, 0, 0, None, 0, 0, None, 0, 0, None, 0, None, 0, 0, 0, 1.0, 0, 0, None, 0, None) == 1
    assert lib.vdb_attention_dk_pad(40) == 64 and lib.vdb_attention_dv_pad(40) == 48
    assert lib.vdb_attention_dk_pad(160) == 192 and lib.vdb_attention_dv_pad(160) == 160
    assert lib.vdb_attention_dk_pad(512) == -1


def test_misaligned_output_or_residual_is_rejected_before_launch():
    """A bf16 `out` or `resid` that is not 16-byte aligned fails the TMA-store tensor map, and the launch would fall back to the
    epilogues that store and load 16-byte vectors there: the entry points refuse such pointers up front (the fake addresses
    below are never dereferenced)."""
    from vdb200._lib import lib
    A, W, ok, bad = 0x10000, 0x20000, 0x30000, 0x30008
    gemm = lambda out, resid: lib.vdb_gemm_bf16(A, 256, 64, 64, None, 0, 0, W, 64, 64, None, 0, 1, resid, 64 if resid else 0, out, 64,
                                                0, 0, 1.0, 0, 1, None, 0, None)
    for out, resid in ((bad, None), (ok, bad)):
        assert gemm(out, resid) == 1 and b"16-byte aligned" in lib.vdb_last_error()
    assert lib.vdb_conv3x3_bf16(A, 1, 8, 8, 64, 0, W, 64, 576, None, 0, None, 0, None, 0, None, 0, bad, 64, 0, 0, 0, 1, None, 0,
                                None) == 1 and b"16-byte aligned" in lib.vdb_last_error()
    assert lib.vdb_conv3x3_bf16(A, 1, 8, 8, 64, 0, W, 64, 576, None, 0, None, 0, None, 0, bad, 64, ok, 64, 0, 0, 0, 1, None, 0,
                                None) == 1 and b"16-byte aligned" in lib.vdb_last_error()
    parts = ctypes.c_int(0)
    assert lib.vdb_gemm_ln_bf16(A, 256, 64, 64, W, 64, 64, None, None, 0, bad, 64, 0, None, 0, 0, 0, 0.0, None, 0, None, ok,
                                ctypes.byref(parts), 0, None) == 1 and b"16-byte aligned" in lib.vdb_last_error()


def test_attention_dispatch_edges():
    """The instantiation table test_attention_coverage_gpu restates: the pads at each band's edges, and the d_head values
    between and above the bands refused with VDB_ERR_UNSUPPORTED by both entry points before any launch (the fake
    addresses below are never dereferenced)."""
    from vdb200._lib import lib
    pads = {8: (64, 48), 48: (64, 48), 56: (64, 64), 64: (64, 64), 72: (128, 80), 80: (128, 80), 136: (192, 160), 160: (192, 160)}
    for d, want in pads.items():
        assert (lib.vdb_attention_dk_pad(d), lib.vdb_attention_dv_pad(d)) == want, d
    Q, K, Vt, out, kv_len = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    before = lib.vdb_launch_count()
    for d in (88, 96, 128, 168, 200):
        assert lib.vdb_attention_bf16(Q, 2048, 0, K, 2048, 0, Vt, 1024, out, 1024, 2, 2, 128, 128, 0, 0, d, 0.125, 0, None) == 3, d
        assert b"d_head" in lib.vdb_last_error()
        assert lib.vdb_attention_varlen_bf16(Q, 2048, 0, K, 2048, 0, Vt, 1024, out, 1024, 2, 2, 128, 128, 0, 0, d, 0.125, 0,
                                             kv_len, None) == 3, d
    assert lib.vdb_launch_count() == before


def test_igemm_last_plan_reports_seven_fields():
    from vdb200._lib import lib
    buf = (ctypes.c_int * 7)()
    assert lib.vdb_igemm_last_plan(buf, 7) == 7 and lib.vdb_igemm_last_plan(None, 0) == 7


def test_norm_last_plan_reports_nine_fields_and_refused_calls_leave_it():
    """vdb_norm_last_plan copies at most n fields and returns 9; GroupNorm / LayerNorm / affine calls refused by their
    argument checks launch nothing and leave the record as it was (the fake addresses below are never dereferenced)."""
    from vdb200._lib import lib
    assert lib.vdb_norm_last_plan(None, 0) == 9
    buf = (ctypes.c_int * 9)(*([-7] * 9))
    assert lib.vdb_norm_last_plan(buf, 3) == 9 and list(buf)[3:] == [-7] * 6
    before = (ctypes.c_int * 9)()
    lib.vdb_norm_last_plan(before, 9)
    x, g, b, s, y = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    assert lib.vdb_groupnorm_nhwc(None, 320, None, 0, 2, 64, 32, g, b, 1e-5, 1, s, y, None) == 1
    assert b"groupnorm" in lib.vdb_last_error()
    assert lib.vdb_groupnorm_nhwc(x, 320, None, 0, 2, 64, 32, g, b, 1e-5, 1, None, y, None) == 1
    assert lib.vdb_groupnorm_nhwc(x, 320, None, 0, 1025, 64, 32, g, b, 1e-5, 1, s, y, None) == 3      # batch > 1024
    assert lib.vdb_groupnorm_nhwc(x, 320, None, 0, 2, 64, 16, g, b, 1e-5, 1, s, y, None) == 3         # groups != 32
    assert lib.vdb_groupnorm_nhwc(x, 324, None, 0, 2, 64, 32, g, b, 1e-5, 1, s, y, None) == 3         # C1 % 8
    assert lib.vdb_groupnorm_nhwc(x, 320, x, 12, 2, 64, 32, g, b, 1e-5, 1, s, y, None) == 3           # C2 % 8
    assert lib.vdb_groupnorm_nhwc(x, 4096, x, 32, 2, 64, 32, g, b, 1e-5, 1, s, y, None) == 3          # C / 8 > 512
    assert b"32 groups" in lib.vdb_last_error()
    assert lib.vdb_layernorm(x, 0, 320, g, b, 1e-5, y, None) == 1
    assert lib.vdb_layernorm(None, 4, 320, g, b, 1e-5, y, None) == 1
    assert lib.vdb_layernorm(x, 4, 324, g, b, 1e-5, y, None) == 3
    assert lib.vdb_layernorm(x, 4, 2056, g, b, 1e-5, y, None) == 3 and b"layernorm" in lib.vdb_last_error()
    assert lib.vdb_affine_act_rows(x, 4, 12, g, b, 1, y, None) == 1 and b"affine_act_rows" in lib.vdb_last_error()
    assert lib.vdb_affine_act_rows(x, 0, 16, g, b, 1, y, None) == 1
    after = (ctypes.c_int * 9)()
    lib.vdb_norm_last_plan(after, 9)
    assert list(after) == list(before)


def test_product_path_refuses_cpu_tensors():
    import pytest
    import torch
    from vdb200 import ops
    with pytest.raises(ValueError, match="no CPU fallback"):
        ops.layernorm(torch.zeros(4, 64, dtype=torch.bfloat16), torch.ones(64), torch.zeros(64))
