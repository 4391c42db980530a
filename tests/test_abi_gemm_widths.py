"""CPU tests of the GEMM shape rules behind the recurrent width: the dense-layer GEMMs take any N / No / Ni that is a
multiple of 32 (K stays a multiple of 32), so every Policy width H % 32 == 0 has kernels end to end.  Argument checks run
before any CUDA call, so all of this is testable without a device."""
import pytest

ONE = 4096        # a non-null, 16-byte aligned "pointer": validation rejects the shape before it is ever used


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.mark.parametrize("M", [1, 127, 5000])
def test_gemm_supported_at_multiples_of_32(lib, M):
    assert lib.dc_gemm_tf32x3_supported(M, 96, 64)
    assert lib.dc_gemm_tf32x3_supported(M, 160, 896)
    assert lib.dc_gemm_tf32x3_supported(M, 32, 32)
    assert lib.dc_gemm_tf32x3_supported(M, 128, 128)
    assert not lib.dc_gemm_tf32x3_supported(M, 100, 128)          # N % 32 != 0
    assert not lib.dc_gemm_tf32x3_supported(M, 128, 48)           # K % 32 != 0
    assert not lib.dc_gemm_tf32x3_supported(M, 16, 32)


def test_python_wrappers_follow_the_library(lib):
    from dotaclient_b200 import ops
    assert ops.gemm_tf32x3_supported(300, 96, 64) and not ops.gemm_tf32x3_supported(300, 100, 64)
    assert ops.gemm_wgrad_supported(10, 96, 160) and ops.gemm_wgrad_supported(10, 384, 896)
    assert not ops.gemm_wgrad_supported(10, 100, 128) and not ops.gemm_wgrad_supported(10, 128, 100)
    assert not ops.gemm_wgrad_supported(0, 128, 128)


def test_unsupported_width_is_reported_with_the_rule(lib):
    # forward / data gradient: N = 100 is the pre-rnn layer of a Policy(hidden_size=100)
    assert lib.dc_gemm_tf32x3(ONE, 896, ONE, 896, None, ONE, 100, 64, 100, 896, 0, None) == -2
    assert b"N % 32 == 0 and K % 32 == 0" in lib.dc_last_error()
    assert lib.dc_gemm_tf32x3(ONE, 48, ONE, 48, None, ONE, 128, 64, 128, 48, 0, None) == -2
    # weight gradient
    assert lib.dc_gemm_wgrad_tf32x3(ONE, 100, ONE, 896, 64, 100, 896, ONE, 896, None, 0, ONE, None) == -2
    assert b"No % 32 == 0 and Ni % 32 == 0" in lib.dc_last_error()
    assert lib.dc_gemm_wgrad_tf32x3(ONE, 128, ONE, 100, 64, 128, 100, ONE, 100, None, 0, ONE, None) == -2


@pytest.mark.parametrize("H,cell", [(100, "gru"), (96, "lstm"), (192, "gru"), (4, "lstm")])
def test_policy_of_any_width_constructs_on_cpu(H, cell):
    """No width check in the constructor: a Policy of any width holds and converts a state_dict on the CPU."""
    from dotaclient_b200.policy import Policy
    pol = Policy(hidden_size=H, cell=cell)
    G = 3 if cell == "gru" else 4
    sd = pol.state_dict()
    assert sd["rnn.weight_ih_l0"].shape == (G * H, H) and sd["affine_pre_rnn.weight"].shape == (H, 896)
    assert sd["affine_unit_attention.weight"].shape == (128, H)
    pol2 = Policy(hidden_size=H, cell=cell)
    pol2.load_state_dict(sd)
    assert all(a.equal(b) for a, b in zip(pol2.state_dict().values(), sd.values()))
