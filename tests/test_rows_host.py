"""CPU tests of the argument checks of the row-list entry points (the target-unit head on the tokens of ``dc_target_rows``):
every bad call is refused before any CUDA call, so they run without a GPU."""
import pytest

EINVAL, EUNSUPPORTED = -1, -2
ONE = 4096                                   # any non-null, 16-byte aligned "pointer": validation fails before it is used


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def _refused(lib, rc, code, who):
    assert rc == code, (who, rc)
    assert who.encode() in lib.dc_last_error(), lib.dc_last_error()


def test_gemm_rows_argument_errors(lib):
    def call(A=ONE, B=ONE, bias=None, C=ONE, C_rows=ONE, ldc=128, M=100, count=ONE, rows=ONE, gather=1, N=128, K=128):
        return lib.dc_gemm_tf32x3_rows(A, K, B, K, bias, C, C_rows, ldc, M, count, rows, gather, N, K, 0, None)

    who = "dc_gemm_tf32x3_rows"
    _refused(lib, call(count=None), EINVAL, who)                   # the count lives on the device and must be given
    _refused(lib, call(C=None, C_rows=None), EINVAL, who)          # nothing to write
    _refused(lib, call(rows=None), EINVAL, who)                    # gather_a without rows
    _refused(lib, call(rows=None, gather=0), EINVAL, who)          # C_rows without rows
    _refused(lib, call(A=None), EINVAL, who)
    _refused(lib, call(B=None), EINVAL, who)
    _refused(lib, call(C_rows=ONE + 4), EINVAL, who)               # misaligned C_rows
    _refused(lib, call(C_rows=None, C=ONE + 8), EINVAL, who)       # misaligned C
    _refused(lib, call(bias=ONE + 4), EINVAL, who)
    _refused(lib, call(N=100), EUNSUPPORTED, who)                  # N % 32
    _refused(lib, call(K=100), EUNSUPPORTED, who)                  # K % 32
    _refused(lib, call(M=0), EUNSUPPORTED, who)                    # M sizes the grid: at least one row
    _refused(lib, call(ldc=96), EINVAL, who)                       # pitch below N
    _refused(lib, call(ldc=130), EINVAL, who)                      # pitch not a multiple of 4


def test_wgrad_rows_argument_errors(lib):
    def call(dy=ONE, X=ONE, x_rows=ONE, T=100, t_dev=ONE, No=128, Ni=128, dW=ONE, db=ONE, ws=ONE):
        return lib.dc_gemm_wgrad_tf32x3_rows(dy, No, X, Ni, x_rows, T, t_dev, No, Ni, dW, Ni, db, 0, ws, None)

    who = "dc_gemm_wgrad_tf32x3_rows"
    _refused(lib, call(t_dev=None), EINVAL, who)
    _refused(lib, call(dy=None), EINVAL, who)
    _refused(lib, call(X=None), EINVAL, who)
    _refused(lib, call(dW=None), EINVAL, who)
    _refused(lib, call(ws=None), EINVAL, who)
    _refused(lib, call(No=100), EUNSUPPORTED, who)                 # No % 32
    _refused(lib, call(Ni=100), EUNSUPPORTED, who)                 # Ni % 32
    _refused(lib, call(T=0), EUNSUPPORTED, who)                    # T sizes the token range: at least one row
    _refused(lib, call(X=ONE + 4), EINVAL, who)
    _refused(lib, call(db=ONE + 8), EINVAL, who)


@pytest.mark.parametrize("fwd", [True, False])
def test_head_rows_argument_errors(lib, fwd):
    from dotaclient_b200 import _lib
    good = (_lib._c.c_void_p * 6)(*([ONE] * 6))
    null5 = (_lib._c.c_void_p * 6)(*([ONE] * 5 + [None]))

    def call(src=ONE, units=good, out=ONE, ld=896, N=8, rows=ONE, count=ONE):
        if fwd:
            return lib.dc_target_unit_q_fwd_rows(src, ld, units, ONE, ONE, out, N, rows, count, None)
        return lib.dc_target_unit_q_bwd_rows(src, units, ONE, ONE, out, ld, N, rows, count, None)

    who = "dc_target_unit_q_fwd_rows" if fwd else "dc_target_unit_q_bwd_rows"
    _refused(lib, call(rows=None), EINVAL, who)
    _refused(lib, call(count=None), EINVAL, who)
    _refused(lib, call(src=None), EINVAL, who)
    _refused(lib, call(out=None), EINVAL, who)
    _refused(lib, call(units=null5), EINVAL, who)
    _refused(lib, call(N=0), EINVAL, who)
    _refused(lib, call(ld=640), EINVAL, who)                       # q / s narrower than 896
    _refused(lib, call(ld=898), EINVAL, who)                       # pitch not a multiple of 4
    if fwd:
        _refused(lib, call(src=ONE + 4), EINVAL, who)              # misaligned q
    else:
        _refused(lib, call(out=ONE + 4), EINVAL, who)              # misaligned s


def test_target_rows_argument_errors(lib):
    def call(mask=ONE, action=ONE, N=100, rows=ONE, count=ONE, flags=ONE, ws=ONE):
        return lib.dc_target_rows(mask, action, N, rows, count, flags, ws, None)

    who = "dc_target_rows"
    _refused(lib, call(N=0), EINVAL, who)
    _refused(lib, call(N=-1), EINVAL, who)
    _refused(lib, call(mask=None), EINVAL, who)
    _refused(lib, call(action=None), EINVAL, who)
    _refused(lib, call(rows=None), EINVAL, who)
    _refused(lib, call(count=None), EINVAL, who)
    _refused(lib, call(flags=None), EINVAL, who)
    _refused(lib, call(ws=None), EINVAL, who)
    _refused(lib, call(mask=ONE + 4), EINVAL, who)                 # rows are read as 8-byte words
    _refused(lib, call(action=ONE + 44), EINVAL, who)              # one 40-byte row and 4 bytes in
    _refused(lib, call(flags=ONE + 2), EINVAL, who)
    assert lib.dc_target_rows_workspace_bytes(0) == 0
    assert lib.dc_target_rows_workspace_bytes(1) == 4 and lib.dc_target_rows_workspace_bytes(1025) == 8


def test_rows_zero_inactive_argument_errors(lib):
    def call(flags=ONE, N=100, dst=ONE, ld=128, width=128):
        return lib.dc_rows_zero_inactive(flags, N, dst, ld, width, None)

    who = "dc_rows_zero_inactive"
    _refused(lib, call(width=126), EINVAL, who)                    # width % 4
    _refused(lib, call(width=0), EINVAL, who)
    _refused(lib, call(ld=124), EINVAL, who)                       # ld < width
    _refused(lib, call(ld=130, width=128), EINVAL, who)            # ld % 4
    _refused(lib, call(N=0), EINVAL, who)
    _refused(lib, call(flags=None), EINVAL, who)
    _refused(lib, call(dst=None), EINVAL, who)
    _refused(lib, call(dst=ONE + 8), EINVAL, who)                  # rows are zeroed as 16-byte words
