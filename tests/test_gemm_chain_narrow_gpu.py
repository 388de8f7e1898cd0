"""A chain link whose last 256-column tile holds <= 128 real columns (N = 640, 1920: the C640 transformer level's
to_out / ff.net.2 / to_qkv) runs that tile 256 wide over the weight box's zero fill, where a single launch runs a
128-column unit.  Both must give the same bits: same outputs, same LayerNorm row statistics."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from diffsensei_b200 import ops as o
    return o


@pytest.mark.parametrize("N,K", [(640, 640), (640, 2560), (1920, 640)])
@pytest.mark.parametrize("M", [4096, 128 * 9 + 40])
def test_chain_link_with_narrow_last_tile_matches_single_launch(ops, M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    r = lambda *s: torch.randn(*s, device=DEV, generator=g)
    a, w, b = r(M, K).to(bf16), (r(N, K) * K ** -0.5).to(bf16), r(N)
    res = r(M, N).to(bf16)
    lns = torch.stack([a.float().sum(1), a.float().pow(2).sum(1)], 1).double().flatten().contiguous()
    colsum = r(N)
    variants = [dict(), dict(residual=res), dict(ln_stats=lns, ln_colsum=colsum), dict(epilogue=ops.EPI_GELU)]
    for kw in variants:
        want = ops.gemm(a, w, b, **kw)
        got = ops.gemm_chain([((a, w, b), kw)], min_links=1)[0]
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"output differs for {sorted(kw)}"
    st_want = torch.zeros(2 * M, dtype=torch.float64, device=DEV)
    st_got = torch.zeros(2 * M, dtype=torch.float64, device=DEV)
    want = ops.gemm(a, w, b, residual=res, row_stats_out=st_want)
    got = ops.gemm_chain([((a, w, b), dict(residual=res, row_stats_out=st_got))], min_links=1)[0]
    torch.cuda.synchronize()
    assert torch.equal(got, want) and torch.equal(st_got, st_want)
