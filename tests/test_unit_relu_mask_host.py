"""CPU tests of the argument checks of the unit encoder's ReLU-mask entry points (dc_unit_embed_fwd_mask stores the mask,
dc_unit_dgrad_fused_mask reads it): every bad call is refused before any CUDA call, so they run without a GPU."""
import pytest


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_unit_embed_fwd_mask_argument_errors(lib):
    assert lib.dc_version() >= 108
    one = 4096                                       # any non-null, 16-byte aligned "pointer": validation fails before it is used

    def call(units=one, mask=one, w=one, ld=896, am=one, n=8, nu=16):
        return lib.dc_unit_embed_fwd_mask(units, one, one, None, mask, w, one, one, None, ld, am, n, nu, None)

    assert call(units=None) == -1 and b"dc_unit_embed_fwd" in lib.dc_last_error()
    assert call(w=None) == -1
    assert call(n=0) == -1
    assert call(nu=4) == -2                          # 1, 5 or 16 units
    assert call(am=None) == -1                       # the max-pool needs its arg-max
    assert call(ld=898) == -1
    assert call(mask=one + 4) == -1                  # the mask rows are 16 bytes, read as one 16-byte load
    assert b"mask_out" in lib.dc_last_error()


def test_unit_dgrad_fused_mask_argument_errors(lib):
    one = 4096

    def call(dx=one, am=one, dl=None, att=None, w_t=one, units=one, mask=one, nu=16, ws=one):
        return lib.dc_unit_dgrad_fused_mask(dx, None, 896, am, dl, 40, att, w_t, units, mask, one, one, 8, nu, one, one, 0, ws, None)

    assert call(w_t=None) == -1 and b"dc_unit_dgrad_fused" in lib.dc_last_error()
    assert call(ws=None) == -1
    assert call(nu=4) == -2                          # 1, 5 or 16
    assert call(am=None) == -1                       # routing without arg-max
    assert call(dl=one) == -1                        # dlogits without att
    assert call(units=one + 4) == -1
    assert call(mask=one + 4) == -1                  # misaligned mask
    assert b"mask" in lib.dc_last_error()
