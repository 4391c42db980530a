"""Weight-gradient GEMM (dc_gemm_wgrad_tf32x3, dc_unit_wgrad_routed) at token counts where every CTA wraps the operand ring
many times: plain dW = dY^T X with dY as a strided column view and accumulation into an existing gradient, and the routed
form of the 5- and 16-unit groups with a last chunk of fewer tokens than a chunk holds.  Checked against float64 with the
3xTF32 bound 3e-6 * sum |dY||X|, and bitwise against a repeated call (the split-K reduction has a fixed order)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _bound(a, b):
    return 3e-6 * (a.double().abs().t() @ b.double().abs()).max().item()


@pytest.mark.parametrize("T,No,Ni,ld,accumulate", [(300001, 128, 128, 128, False), (300001, 512, 128, 512, False),
                                                   (300001, 128, 896, 896, True), (300001, 96, 160, 896, True),
                                                   (300001, 128, 128, 896, False)])
def test_plain_wgrad_long_ring(T, No, Ni, ld, accumulate):
    """dW (+)= dY^T X, db = colsum dY; ld > No: dY is the column slice [:, 64:64+No] of a [T, ld] buffer (row pitch ld)."""
    from dotaclient_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(T + No + Ni + ld)
    buf = torch.randn(T, max(ld, No + 64) if ld > No else No, generator=g, device=DEV)
    dy = buf[:, 64:64 + No] if ld > No else buf
    x = torch.randn(T, Ni, generator=g, device=DEV)
    base, base_b = torch.randn(No, Ni, generator=g, device=DEV), torch.randn(No, generator=g, device=DEV)

    def run():
        dw = base.clone() if accumulate else torch.full((No, Ni), 7.0, device=DEV)
        db = base_b.clone() if accumulate else torch.full((No,), 7.0, device=DEV)
        return ops.gemm_wgrad_tf32x3(dy, x, dw_out=dw, db_out=db, accumulate=accumulate)

    dw, db = run()
    ref = dy.double().t() @ x.double() + (base.double() if accumulate else 0.0)
    assert (dw.double() - ref).abs().max().item() <= _bound(dy, x) + (1e-6 * base.abs().max().item() if accumulate else 0.0)
    refb = dy.double().sum(0) + (base_b.double() if accumulate else 0.0)
    assert (db.double() - refb).abs().max().item() <= 1e-6 * (dy.double().abs().sum(0).max().item() + 1.0)
    dw2, db2 = run()
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


@pytest.mark.parametrize("N,n_u,dx2", [(18751, 16, True), (18751, 16, False), (60001, 5, True), (60001, 5, False)])
def test_routed_wgrad_long_ring(N, n_u, dx2):
    """dW = R^T basic, db = colsum R, R[(n,u), c] = (argmax[n,c] == u) ? d_xmax[n,c] (+ d_xmax2[n,c]) : 0 with d_xmax and
    d_xmax2 column slices of a [N, 896] buffer; N is odd (16 units: 2 tokens per chunk) and N % 6 != 0 (5 units: 6)."""
    from dotaclient_b200 import _lib
    lib, st = _lib.load(), _lib.stream_ptr()
    g = torch.Generator(device=DEV).manual_seed(N * n_u)
    xcat = torch.randn(N, 896, generator=g, device=DEV)
    am = torch.randint(0, n_u, (N, 128), generator=g, device=DEV, dtype=torch.uint8)
    basic = torch.randn(N * n_u, 128, generator=g, device=DEV)
    d = xcat[:, 256:384] + (xcat[:, 640:768] if dx2 else 0.0)
    R = torch.where(am.long().unsqueeze(1) == torch.arange(n_u, device=DEV).view(1, n_u, 1), d.unsqueeze(1), 0.0).reshape(N * n_u, 128)
    ws = torch.empty(int(lib.dc_gemm_wgrad_workspace_bytes(128, 128)), dtype=torch.uint8, device=DEV)
    out = []
    for _ in range(2):
        dW, db = torch.full((128, 128), 7.0, device=DEV), torch.full((128,), 7.0, device=DEV)
        p = xcat.data_ptr()
        _lib.check(lib.dc_unit_wgrad_routed(p + 4 * 256, p + 4 * 640 if dx2 else None, 896, am.data_ptr(), basic.data_ptr(), N, n_u,
                                            dW.data_ptr(), db.data_ptr(), ws.data_ptr(), st), "dc_unit_wgrad_routed")
        out.append((dW, db))
    (dW, db), (dW2, db2) = out
    assert (dW.double() - R.double().t() @ basic.double()).abs().max().item() <= _bound(R, basic)
    assert (db.double() - R.double().sum(0)).abs().max().item() <= 1e-6 * R.double().abs().sum(0).max().item()
    assert torch.equal(dW, dW2) and torch.equal(db, db2)
