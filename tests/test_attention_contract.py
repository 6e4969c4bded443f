"""The host checks of the attention entry points refuse, before any launch and before any tensor map is made, descriptors
their kernels cannot address, and name the violated constraint (no GPU needed: the fake pointers below are never
dereferenced). Both kernel families are covered: the wgmma kernels (attention.cu, inner == 1 or S > 32) and the
short-sequence kernels (attention_small.cu, inner > 1 and S <= 32)."""
import ctypes

import pytest

P = 1024            # a 16-byte aligned fake device pointer
HEADS = 5
C = HEADS * 64


@pytest.fixture(scope="module")
def lib():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200 import _lib
    return _lib.load()


def _rejects(lib, rc, msg):
    assert rc == -1, rc
    assert lib.svdx_last_error().decode() == msg


# (S, nseq, inner, outer_stride, inner_stride, tok_stride) of each family
WGMMA = dict(S=144, nseq=2, inner=1, outer_stride=144, inner_stride=0, tok_stride=1)
WGMMA_STRIDED = dict(S=40, nseq=6, inner=3, outer_stride=120, inner_stride=1, tok_stride=3)
SMALL = dict(S=14, nseq=6, inner=3, outer_stride=42, inner_stride=1, tok_stride=3)


def _desc(geo, **kw):
    from svd_xtend_b200._lib import SvdxAttn
    d = SvdxAttn()
    d.q = d.k = d.v = d.o = d.dout = d.dq = d.dk = d.dv = d.lse = d.delta = P
    d.ldq = d.ldk = d.ldv = d.ldo = d.lddo = d.lddq = d.lddk = d.lddv = 3 * C
    d.heads, d.scale = HEADS, 0.125
    for n, v in {**geo, **kw}.items():
        setattr(d, n, v)
    return d


def _fwd(lib, geo, **kw):
    return lib.svdx_attention_fwd(ctypes.byref(_desc(geo, **kw)), None)


def _bwd(lib, geo, **kw):
    return lib.svdx_attention_bwd(ctypes.byref(_desc(geo, **kw)), None)


@pytest.mark.parametrize("geo", [WGMMA, WGMMA_STRIDED], ids=["dense", "strided"])
def test_wgmma_refuses_null_pointers(lib, geo):
    for n in ("q", "k", "v"):
        _rejects(lib, _fwd(lib, geo, **{n: None}), "attention: null pointer")
        _rejects(lib, _bwd(lib, geo, **{n: None}), "attention: null pointer")
    _rejects(lib, _fwd(lib, geo, o=None), "attention_fwd: output")
    for n in ("o", "dout", "dq", "dk", "dv", "lse", "delta"):
        _rejects(lib, _bwd(lib, geo, **{n: None}), "attention_bwd: null pointer")


def test_small_refuses_null_pointers(lib):
    for n in ("q", "k", "v", "o"):
        _rejects(lib, _fwd(lib, SMALL, **{n: None}), "attention(small): null pointer")
    for n in ("dout", "dq", "dk", "dv"):
        _rejects(lib, _bwd(lib, SMALL, **{n: None}), "attention_bwd(small): null pointer")


def test_sequence_geometry(lib):
    _rejects(lib, _fwd(lib, WGMMA_STRIDED, nseq=7), "attention: bad sequence geometry")
    _rejects(lib, _bwd(lib, WGMMA_STRIDED, nseq=7), "attention: bad sequence geometry")
    _rejects(lib, _fwd(lib, SMALL, nseq=7), "attention(small): bad sequence geometry")
    _rejects(lib, _bwd(lib, SMALL, nseq=7), "attention(small): bad sequence geometry")
    for S in (129, 256):
        _rejects(lib, _fwd(lib, WGMMA_STRIDED, S=S), "attention: strided sequences longer than 128 tokens are not supported")
        _rejects(lib, _bwd(lib, WGMMA_STRIDED, S=S), "attention: strided sequences longer than 128 tokens are not supported")


@pytest.mark.parametrize("geo", [WGMMA, WGMMA_STRIDED], ids=["dense", "strided"])
def test_wgmma_leading_dims(lib, geo):
    for n in ("ldq", "ldk", "ldv"):
        _rejects(lib, _fwd(lib, geo, **{n: 3 * C + 4}), "attention: leading dims must be multiples of 8")
        _rejects(lib, _fwd(lib, geo, **{n: C - 8}), "attention: ldq / ldk / ldv < heads * 64")
        _rejects(lib, _bwd(lib, geo, **{n: C - 8}), "attention: ldq / ldk / ldv < heads * 64")
    _rejects(lib, _fwd(lib, geo, ldo=C + 4), "attention_fwd: output")
    _rejects(lib, _fwd(lib, geo, ldo=C - 8), "attention_fwd: ldo < heads * 64")
    for n in ("ldo", "lddo", "lddq", "lddk", "lddv"):
        _rejects(lib, _bwd(lib, geo, **{n: C + 4}), "attention_bwd: leading dims")
        _rejects(lib, _bwd(lib, geo, **{n: C - 8}), "attention_bwd: ldo / lddo / lddq / lddk / lddv < heads * 64")


def test_small_leading_dims(lib):
    for n in ("ldq", "ldk", "ldv", "ldo"):
        _rejects(lib, _fwd(lib, SMALL, **{n: C + 4}), "attention(small): leading dims must be multiples of 8")
        _rejects(lib, _fwd(lib, SMALL, **{n: C - 8}), "attention(small): ldq / ldk / ldv / ldo < heads * 64")
        _rejects(lib, _bwd(lib, SMALL, **{n: C - 8}), "attention(small): ldq / ldk / ldv / ldo < heads * 64")
    for n in ("lddo", "lddq", "lddk", "lddv"):
        _rejects(lib, _bwd(lib, SMALL, **{n: C + 4}), "attention_bwd(small): leading dims")
        _rejects(lib, _bwd(lib, SMALL, **{n: C - 8}), "attention_bwd(small): lddo / lddq / lddk / lddv < heads * 64")


@pytest.mark.parametrize("geo", [WGMMA, WGMMA_STRIDED], ids=["dense", "strided"])
def test_wgmma_output_alignment(lib, geo):
    # the outputs are stored as 4-byte column pairs
    _rejects(lib, _fwd(lib, geo, o=P + 2), "attention: o / dq / dk / dv must be 4 B aligned")
    for n in ("o", "dq", "dk", "dv"):
        _rejects(lib, _bwd(lib, geo, **{n: P + 2}), "attention: o / dq / dk / dv must be 4 B aligned")


def test_small_operand_alignment(lib):
    # the short-sequence kernels move whole 16-byte pieces of every row
    for n in ("q", "k", "v", "o"):
        _rejects(lib, _fwd(lib, SMALL, **{n: P + 8}), "attention(small): operands must be 16 B aligned")
    for n in ("dout", "dq", "dk", "dv"):
        _rejects(lib, _bwd(lib, SMALL, **{n: P + 8}), "attention_bwd(small): operands must be 16 B aligned")


def _hd80(lib, q=P, ldq=3 * 1280, ldk=3 * 1280, ldv=3 * 1280, o=P, ldo=1280, heads=16, S=257, nseq=2):
    return lib.svdx_attention_hd80_fwd(q, ldq, P, ldk, P, ldv, o, ldo, nseq, heads, S, 0.125, None)


def test_hd80_checks(lib):
    msg = "attention_hd80_fwd: q/k/v rows need ld % 8 == 0 and ld >= heads * 80, o rows ld even"
    for n in ("ldq", "ldk", "ldv", "ldo"):
        _rejects(lib, _hd80(lib, **{n: 1280 - 8}), msg)
    _rejects(lib, _hd80(lib, ldq=3 * 1280 + 4), msg)
    _rejects(lib, _hd80(lib, ldo=1281), msg)
    _rejects(lib, _hd80(lib, q=P + 8), "attention_hd80_fwd: q/k/v 16 B and o 4 B aligned")
    _rejects(lib, _hd80(lib, o=P + 2), "attention_hd80_fwd: q/k/v 16 B and o 4 B aligned")
    _rejects(lib, _hd80(lib, q=None), "attention_hd80_fwd: null pointer or bad geometry")
