"""CPU tests of the argument checks of the fused unit-embedding forward and of the target-unit head on raw unit features:
every bad call is refused before any CUDA call, so they run without a GPU."""
import pytest


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_unit_embed_fwd_argument_errors(lib):
    assert lib.dc_version() >= 106
    one = 4096                                       # any non-null, 16-byte aligned "pointer": validation fails before it is used

    def call(units=one, w_b=one, b_b=one, basic=None, w=one, bias=one, xmax=one, copy=None, ld=896, am=one, n=8, nu=16):
        return lib.dc_unit_embed_fwd(units, w_b, b_b, basic, w, bias, xmax, copy, ld, am, n, nu, None)

    assert call(units=None) == -1 and b"dc_unit_embed_fwd" in lib.dc_last_error()
    assert call(w_b=None) == -1
    assert call(xmax=None) == -1
    assert call(n=0) == -1
    assert call(nu=4) == -2                          # 1, 5 or 16 units
    assert call(am=None) == -1                       # the max-pool needs its arg-max
    assert call(nu=1) == -1                          # ... and a 1-unit group has none
    assert call(nu=1, am=None, copy=one) == -1
    assert call(ld=64) == -1                         # row pitch below 128
    assert call(ld=898) == -1                        # row pitch not a multiple of 4
    assert call(units=one + 4) == -1                 # misaligned operands
    assert call(basic=one + 8) == -1
    assert call(xmax=one + 4) == -1
    assert b"dc_unit_embed_fwd" in lib.dc_last_error()


def test_target_unit_head_argument_errors(lib):
    from dotaclient_b200 import _lib
    one = 4096
    good = (_lib._c.c_void_p * 6)(*([one] * 6))
    null5 = (_lib._c.c_void_p * 6)(*([one] * 5 + [None]))
    skew = (_lib._c.c_void_p * 6)(*([one] * 2 + [one + 4] + [one] * 3))
    for units in (null5, skew):                      # a missing or misaligned unit array
        assert lib.dc_target_unit_q_fwd(one, 896, units, one, one, one, 8, None) == -1
        assert b"dc_target_unit_q_fwd" in lib.dc_last_error()
        assert lib.dc_target_unit_q_bwd(one, units, one, one, one, 896, 8, None) == -1
        assert b"dc_target_unit_q_bwd" in lib.dc_last_error()
    assert lib.dc_target_unit_q_fwd(one, 896, good, None, one, one, 8, None) == -1      # no W_b
    assert lib.dc_target_unit_q_bwd(one, good, one, None, one, 896, 8, None) == -1      # no b_b
    assert lib.dc_target_unit_q_fwd(one, 640, good, one, one, one, 8, None) == -1       # q narrower than 896
