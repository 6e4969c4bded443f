"""The host checks of the elementwise / layout / reduction entry points refuse, before any launch, arguments their kernels
cannot address, and name the violated constraint (no GPU needed: the fake pointers below are never dereferenced)."""
import ctypes

import pytest
import torch

P = 1024            # a 16-byte aligned fake device pointer
P8 = 1032           # 8-byte aligned, not 16
P4 = 1028           # 4-byte aligned


@pytest.fixture(scope="module")
def lib():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200 import _lib
    return _lib.load()


def _rejects(lib, rc, msg):
    assert rc == -1, rc
    assert lib.svdx_last_error().decode() == msg


def test_colsum_checks_the_row_stride(lib):
    _rejects(lib, lib.svdx_colsum(P, 8, 2, 16, P, 0, None), "colsum: ldx < cols")


def test_geglu_bwd_checks_alignment_and_row_strides(lib):
    msg = "geglu_bwd: pre, dout and dpre must be 16-byte aligned"
    _rejects(lib, lib.svdx_geglu_bwd(P8, 32, P, 16, P, 32, 2, 16, None, None), msg)
    _rejects(lib, lib.svdx_geglu_bwd(P, 32, P8, 16, P, 32, 2, 16, None, None), msg)
    _rejects(lib, lib.svdx_geglu_bwd(P, 32, P, 16, P8, 32, 2, 16, P, None), msg)
    _rejects(lib, lib.svdx_geglu_bwd(P, 24, P, 16, P, 32, 2, 16, P, None), "geglu_bwd: ldpre < 2h")
    _rejects(lib, lib.svdx_geglu_bwd(P, 32, P, 8, P, 32, 2, 16, None, None), "geglu_bwd: lddo < h")
    _rejects(lib, lib.svdx_geglu_bwd(P, 32, P, 16, P, 16, 2, 16, P, None), "geglu_bwd: lddpre < 2h")


def test_softmax_rows_checks_both_row_strides(lib):
    _rejects(lib, lib.svdx_softmax_rows(P, 8, 2, 16, 1.0, P, 16, None), "softmax_rows: ldx < cols")
    _rejects(lib, lib.svdx_softmax_rows(P, 16, 2, 16, 1.0, P, 8, None), "softmax_rows: ldy < cols")


def test_gemv_checks_every_row_stride(lib):
    from svd_xtend_b200._lib import OUT_BF16, OUT_F32
    _rejects(lib, lib.svdx_gemv(P, 8, P, 16, 2, 4, 16, None, P, 4, OUT_BF16, 1.0, 0, None), "gemv: lda < K")
    _rejects(lib, lib.svdx_gemv(P, 16, P, 8, 2, 4, 16, None, P, 4, OUT_F32, 1.0, 0, None), "gemv: ldw < K")
    _rejects(lib, lib.svdx_gemv(P, 16, P, 16, 2, 4, 16, None, P, 3, OUT_F32, 1.0, 1, None), "gemv: ldo < N")


def test_outer_accum_checks_every_row_stride(lib):
    _rejects(lib, lib.svdx_outer_accum(P, 4, P, 8, 2, 8, 8, None, P, 8, None), "outer_accum: lddy < O")
    _rejects(lib, lib.svdx_outer_accum(P, 8, P, 4, 2, 8, 8, None, P, 8, None), "outer_accum: ldx < K")
    _rejects(lib, lib.svdx_outer_accum(P, 8, P, 8, 2, 8, 8, None, P, 4, None), "outer_accum: ldg < K")


def test_dot_diff_checks_alignment(lib):
    msg = "dot_diff: dy, a and b must be 16-byte aligned"
    for dy, a, b in ((P8, P, P), (P, P8, P), (P, P, P8)):
        _rejects(lib, lib.svdx_dot_diff(dy, a, b, 64, P, None), msg)


def test_splitk_epilogue_checks_alignment_and_row_strides(lib):
    def call(ws=P, ldw=16, out=P, ldo=16, rowbias=None, ldrb=0, res1=None, ldr1=0, res2=None, ldr2=0):
        return lib.svdx_splitk_epilogue(ws, ldw, out, ldo, 2, 16, None, rowbias, 1, ldrb, res1, ldr1, res2, ldr2, None, None)
    _rejects(lib, call(ws=P4), "splitk_epilogue: ws must be 16-byte aligned")
    msg = "splitk_epilogue: out, res1 and res2 must be 16-byte aligned"
    _rejects(lib, call(out=P8), msg)
    _rejects(lib, call(res1=P8, ldr1=16), msg)
    _rejects(lib, call(res2=P8, ldr2=16), msg)
    _rejects(lib, call(ldw=8), "splitk_epilogue: ldw < cols")
    _rejects(lib, call(ldo=8), "splitk_epilogue: ldo < cols")
    _rejects(lib, call(res1=P, ldr1=8), "splitk_epilogue: ldr1 < cols")
    _rejects(lib, call(res2=P, ldr2=8), "splitk_epilogue: ldr2 < cols")
    _rejects(lib, call(rowbias=P, ldrb=8), "splitk_epilogue: ldrb < cols")


# ---- the Python wrappers index their operands as flat bf16 arrays: anything else is refused before the library is reached
def _bf(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def test_concat_channels_refuses_what_it_cannot_index():
    from svd_xtend_b200 import raw
    with pytest.raises(ValueError, match="concat_channels: b must be bfloat16"):
        raw.concat_channels(_bf(4, 8), torch.zeros(4, 8), _bf(4, 16))
    with pytest.raises(ValueError, match="concat_channels: dst must be contiguous"):
        raw.concat_channels(_bf(4, 8), _bf(4, 8), _bf(4, 32)[:, :16])
    with pytest.raises(ValueError, match="concat_channels: operands must have the same row count"):
        raw.concat_channels(_bf(4, 8), _bf(5, 8), _bf(4, 16))
    with pytest.raises(ValueError, match="concat_channels: dst has 24 channels"):
        raw.concat_channels(_bf(4, 8), _bf(4, 8), _bf(4, 24))


def test_split_channels_refuses_what_it_cannot_index():
    from svd_xtend_b200 import raw
    with pytest.raises(ValueError, match="split_channels: src must be bfloat16"):
        raw.split_channels(torch.zeros(4, 16, dtype=torch.float16), _bf(4, 8), _bf(4, 8))
    with pytest.raises(ValueError, match="split_channels: a must be contiguous"):
        raw.split_channels(_bf(4, 16), _bf(8, 8)[::2], _bf(4, 8))
    with pytest.raises(ValueError, match="split_channels: operands must have the same row count"):
        raw.split_channels(_bf(4, 16), _bf(3, 8), None)
    with pytest.raises(ValueError, match="split_channels: operands must have the same row count"):
        raw.split_channels(_bf(4, 16), _bf(4, 8), _bf(2, 8))
    with pytest.raises(ValueError, match="split_channels: src has 16 channels"):
        raw.split_channels(_bf(4, 16), _bf(4, 8), _bf(4, 16))


def test_axpby_refuses_what_it_cannot_index():
    from svd_xtend_b200 import raw
    with pytest.raises(ValueError, match="axpby: y must be bfloat16"):
        raw.axpby(_bf(64), _bf(64), torch.zeros(64))
    with pytest.raises(ValueError, match="axpby: a must be contiguous"):
        raw.axpby(_bf(8, 16)[:, :8], _bf(64), _bf(64))
    with pytest.raises(ValueError, match="axpby: a, b and y must have the same length"):
        raw.axpby(_bf(64), _bf(64), _bf(56))
    with pytest.raises(ValueError, match="axpby: scales must be fp32 with at least 2 elements"):
        raw.axpby(_bf(64), _bf(64), _bf(64), torch.zeros(1))
    with pytest.raises(ValueError, match="axpby: scales must be fp32 with at least 2 elements"):
        raw.axpby(_bf(64), _bf(64), _bf(64), torch.zeros(2, dtype=torch.float64))
