"""The host checks of the GroupNorm and LayerNorm entry points refuse, before any launch, row strides their kernels would
use to read or write into the neighbouring rows, and name the violated constraint (no GPU needed: the fake pointers below
are never dereferenced)."""
import pytest

P = 1024            # a 16-byte aligned fake device pointer
C1, C2 = 256, 64    # two sources of a 320-channel GroupNorm (32 groups of 10 channels)
C = C1 + C2
OUTER, ROWS = 2, 16


@pytest.fixture(scope="module")
def lib():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200 import _lib
    return _lib.load()


def _rejects(lib, rc, msg):
    assert rc == -1, rc
    assert lib.svdx_last_error().decode() == msg


def _gn_sums(lib, ldx=C, ldx2=C, outer=OUTER, rows=ROWS):
    return lib.svdx_groupnorm_sums(P, ldx, C1, P, ldx2, C2, outer, rows, P, C, None)


def _gn_apply(lib, ldx=C, ldx2=C, ldy=C, outer=OUTER, rows=ROWS):
    return lib.svdx_groupnorm_apply_fused(P, ldx, C1, P, ldx2, C2, outer, rows, 32, 1e-5, P, C, P, C, P, P, P, P, 1, P, ldy, P, None)


def _gn_bwd_sums(lib, ldx=C, ldx2=C, lddy=C, outer=OUTER, rows=ROWS):
    return lib.svdx_groupnorm_bwd_sums(P, ldx, C1, P, ldx2, C2, P, lddy, outer, rows, P, 1, P, None)


def _gn_bwd_fused(lib, ldx=C, ldx2=C, lddy=C, lddx=C, lddx2=C, c2=C2, dres=None, lddres=0, outer=OUTER, rows=ROWS):
    return lib.svdx_groupnorm_bwd_fused(P, ldx, C - c2, P if c2 else None, ldx2, c2, P, lddy, outer, rows, 32, P, P, P, P, 1, P,
                                        P, lddx, P if c2 else None, lddx2, P, P, dres, lddres, None)


@pytest.mark.parametrize("entry", ["groupnorm_sums", "groupnorm_apply_fused", "groupnorm_bwd_sums", "groupnorm_bwd_fused"])
def test_groupnorm_entries_check_the_source_row_strides(lib, entry):
    call = {"groupnorm_sums": _gn_sums, "groupnorm_apply_fused": _gn_apply, "groupnorm_bwd_sums": _gn_bwd_sums,
            "groupnorm_bwd_fused": _gn_bwd_fused}[entry]
    _rejects(lib, call(lib, ldx=C1 - 8), f"{entry}: ldx < C1")
    _rejects(lib, call(lib, ldx2=C2 - 8), f"{entry}: ldx2 < C2")
    # the strides count over all outer * rows rows: two slabs of one row still overlap
    _rejects(lib, call(lib, ldx=C1 - 8, outer=2, rows=1), f"{entry}: ldx < C1")


def test_groupnorm_apply_checks_the_output_row_stride(lib):
    _rejects(lib, _gn_apply(lib, ldy=C - 8), "groupnorm_apply_fused: ldy < C1 + C2")


def test_groupnorm_bwd_sums_checks_the_gradient_row_stride(lib):
    _rejects(lib, _gn_bwd_sums(lib, lddy=C - 8), "groupnorm_bwd_sums: lddy < C")


def test_groupnorm_bwd_fused_checks_every_row_stride(lib):
    _rejects(lib, _gn_bwd_fused(lib, lddy=C - 8), "groupnorm_bwd_fused: lddy < C")
    _rejects(lib, _gn_bwd_fused(lib, lddx=C1 - 8), "groupnorm_bwd_fused: lddx < C1")
    _rejects(lib, _gn_bwd_fused(lib, lddx2=C2 - 8), "groupnorm_bwd_fused: lddx2 < C2")
    # dres is only accepted with a single source, whose dx covers all C channels
    _rejects(lib, _gn_bwd_fused(lib, c2=0, lddx=C, dres=P, lddres=C - 8), "groupnorm_bwd_fused: lddres < C")


def _ln_fwd(lib, ldx=C, ldy=C, addvec=None, ldxs=0, rows=ROWS):
    return lib.svdx_layernorm_fwd(P, ldx, rows, C, P, P, 1e-5, P, ldy, P, P, addvec, 1, P if addvec else None, ldxs, None)


def _ln_bwd(lib, ldx=C, lddy=C, lddx=C, dres=None, lddres=0, rows=ROWS):
    return lib.svdx_layernorm_bwd(P, ldx, P, lddy, rows, C, P, P, P, P, lddx, dres, lddres, P, P, None)


def test_layernorm_fwd_checks_every_row_stride(lib):
    _rejects(lib, _ln_fwd(lib, ldx=C - 8), "layernorm_fwd: ldx < C")
    _rejects(lib, _ln_fwd(lib, ldy=C - 8), "layernorm_fwd: ldy < C")
    _rejects(lib, _ln_fwd(lib, addvec=P, ldxs=C - 8), "layernorm_fwd: ldxs < C")


def test_layernorm_bwd_checks_every_row_stride(lib):
    _rejects(lib, _ln_bwd(lib, ldx=C - 8), "layernorm_bwd: ldx < C")
    _rejects(lib, _ln_bwd(lib, lddy=C - 8), "layernorm_bwd: lddy < C")
    _rejects(lib, _ln_bwd(lib, lddx=C - 8), "layernorm_bwd: lddx < C")
    _rejects(lib, _ln_bwd(lib, dres=P, lddres=C - 8), "layernorm_bwd: lddres < C")
