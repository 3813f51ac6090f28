"""GPU: wgmma building blocks (descriptors, operand layouts, accumulator fragment, BF16x3 split) against a plain fp64 matmul."""
import pytest
import torch

from oracle import grad_check
from pointnerf_b200 import lib as _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(A, W, layout):
    l = _lib.load_selftest()
    K, N = A.shape[1], W.shape[0]
    D = torch.full((128, N), float("nan"), device=DEV)
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check_selftest(l.pnb_umma_selftest(A.data_ptr(), W.data_ptr(), D.data_ptr(), K, N, layout, err.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream), "pnb_umma_selftest")
    torch.cuda.synchronize()
    return D, int(err.item())


@pytest.mark.parametrize("layout", [0, 4])
@pytest.mark.parametrize("K,N", [(16, 16), (32, 256), (64, 128), (288, 256), (272, 256), (256, 256), (100, 64)])
def test_umma_bf16x3_matches_matmul(layout, K, N):
    g = torch.Generator(device=DEV).manual_seed(K * 1000 + N)
    A = torch.randn(128, K, device=DEV, generator=g)
    W = torch.randn(N, K, device=DEV, generator=g) / K ** 0.5
    D, err = _run(A.contiguous(), W.contiguous(), layout)
    assert err == 0, "pipeline timeout code %d" % err
    ref = (A.double() @ W.double().t())
    d = (D.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert d <= 2e-5 * max(scale, 1.0), "layout %d K=%d N=%d: max abs err %.3e (scale %.2f)" % (layout, K, N, d, scale)
    # the split must beat a single bf16 pass by orders of magnitude
    single = (A.bfloat16().double() @ W.bfloat16().double().t() - ref).abs().max().item()
    assert d < single / 50


@pytest.mark.parametrize("layout,K,N", [(100, 16, 16), (100, 64, 256), (100, 256, 256), (101, 32, 256), (101, 272, 256)])
def test_wgmma_a_operand_in_registers(layout, K, N):
    """RS form (A fragments in registers, split into bf16 hi / lo per K step), optionally mixed with one shared-memory K step on the
    same accumulator."""
    g = torch.Generator(device=DEV).manual_seed(K * 7 + N)
    A = torch.randn(128, K, device=DEV, generator=g)
    W = torch.randn(N, K, device=DEV, generator=g) / K ** 0.5
    D, _ = _run(A.contiguous(), W.contiguous(), layout)
    ref = (A.double() @ W.double().t())
    d = (D.double() - ref).abs().max().item()
    assert d <= 2e-5 * max(ref.abs().max().item(), 1.0), "mode %d K=%d N=%d: max abs err %.3e" % (layout, K, N, d)


@pytest.mark.parametrize("mode,K,N", [(0, 32, 256), (0, 288, 256), (0, 64, 64), (1, 16, 32), (1, 256, 256), (1, 64, 128)])
def test_wgmma_cluster_pair(mode, K, N):
    """Cluster of two CTAs (M = 256): each CTA converts half of B and stores it into both CTAs' shared memory (distributed shared
    memory, cluster barriers); A from shared memory (mode 0) or registers (mode 1)."""
    l = _lib.load_selftest()
    g = torch.Generator(device=DEV).manual_seed(K * 13 + N + mode)
    A = torch.randn(256, K, device=DEV, generator=g).contiguous()
    W = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).contiguous()
    D = torch.full((256, N), float("nan"), device=DEV)
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check_selftest(l.pnb_umma_selftest2(A.data_ptr(), W.data_ptr(), D.data_ptr(), K, N, mode, err.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), "pnb_umma_selftest2")
    torch.cuda.synchronize()
    ref = A.double() @ W.double().t()
    d = (D.double() - ref).abs().max().item()
    assert d <= 2e-5 * max(ref.abs().max().item(), 1.0), "mode %d K=%d N=%d: max abs err %.3e" % (mode, K, N, d)


# ---- the wgmma GEMM engine of the backward pass (csrc/gemm_tc.cu) against fp64 matmuls, every operand form it is used in
def _gemm_tc(A, a_rs, a_ks, B, b_rs, b_ks, M, N, K, ldc, bias=None, act=0, dact=None, ldd=0, dact_n=0, splits=1, C0=None, precise=0):
    """C [M x ldc] (C0, or 7.0 everywhere) with 128 guard rows of 7.0 below it that must stay untouched; the split-K workspace starts
    as NaN, so that a partial tile that is not written shows."""
    l = _lib.load_selftest()
    C = torch.full((M + 128, ldc), 7.0, device="cuda")
    if C0 is not None:
        C[:M] = C0
    err = torch.zeros(4, dtype=torch.int32, device="cuda")
    part = torch.full((max(max(splits, 1) * M * N, 1 << 19),), float("nan"), device="cuda")
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check_selftest(l.pnb_gemm_tc_test(A.data_ptr(), a_rs, a_ks, B.data_ptr(), b_rs, b_ks, C.data_ptr(), ldc, M, N, K, ptr(bias), act,
                                           ptr(dact), ldd, dact_n, splits, part.data_ptr(), part.numel() * 4, 1 if C0 is not None else 0,
                                           precise, err.data_ptr(), torch.cuda.current_stream().cuda_stream), "pnb_gemm_tc_test")
    torch.cuda.synchronize()
    assert int(err[0]) == 0
    assert torch.all(C[M:] == 7.0), "rows beyond M written"
    return C[:M]


def _rel(a, ref):
    return ((a.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("M,N,K", [(300, 256, 288), (128, 128, 128), (1000, 256, 272), (77, 288, 256), (4096, 128, 128),
                                   (1000, 256, 512),    # F = 63: the 512-wide block1.0 recompute (its NT: 512 output columns)
                                   # one row, and either side of the 64-row warpgroup half and of the 128-row tile
                                   (1, 256, 288), (2, 256, 272), (63, 128, 128), (64, 256, 288), (65, 128, 272), (127, 288, 256),
                                   (129, 256, 272)])
def test_gemm_tc_nn_nt(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    X = torch.randn(M, K + 16, device="cuda", generator=g)[:, :K]                 # leading dimension != K
    lda = X.stride(0)
    Wt = (0.1 * torch.randn(K, N, device="cuda", generator=g)).contiguous()       # W^T [K][N] as the backward holds the weights
    bias = torch.randn(N, device="cuda", generator=g)
    # NN (forward recompute): H = LeakyReLU(X Wt + b);  A(m,k) = X[m*lda + k], B(n,k) = Wt[k*N + n]
    H = _gemm_tc(X, lda, 1, Wt, 1, N, M, N, K, N + 16, bias=bias, act=1)
    ref = torch.nn.functional.leaky_relu(X.double() @ Wt.double() + bias.double(), 0.01)
    assert _rel(H[:, :N], ref) < 2e-5 and torch.all(H[:, N:] == 7.0)
    # the 3-part split (6 products): stops at ~1e-6 - the tensor core does not accumulate with full fp32 precision.  Its error grows
    # linearly with K, not with M: over M of 1 to 1000 and four seeds, at most 1.2e-6 at K 128, 2.5e-6 at K 256 to 288 and 4.6e-6
    # at K 512 (H100 80GB HBM3, 700 W), so that the bound below holds K 512 on this test's seed of (1000, 256, 512) only
    Hp = _gemm_tc(X, lda, 1, Wt, 1, N, M, N, K, N + 16, bias=bias, act=1, precise=1)
    assert _rel(Hp[:, :N], ref) < 4e-6, _rel(Hp[:, :N], ref)      # ~1e-6: the accumulation precision of the tensor core, not fp32
    # NT (dX = dZ W * LeakyReLU'(Y)): A = dZ [M x N], B(n=k_in, k=n_out) = Wt[k_in*N + n_out]; result [M x K]
    if K % 16 == 0:
        dZ = torch.randn(M, N, device="cuda", generator=g)
        Y = torch.randn(M, K, device="cuda", generator=g)
        dact_n = (K // 16 - 1) * 16
        dX = _gemm_tc(dZ, N, 1, Wt, N, 1, M, K, N, K, dact=Y, ldd=K, dact_n=dact_n)
        refx = dZ.double() @ Wt.double().t()
        mask = torch.where(Y > 0, 1.0, 0.01).double()
        mask[:, dact_n:] = 1.0
        assert _rel(dX, refx * mask) < 2e-5


@pytest.mark.parametrize("dact", [False, True])
def test_gemm_tc_nt_partial_n_tile(dact):
    """The F = 63 dX1 GEMM: 448 of the 512 columns of G1 (the 7F feature inputs rounded up to 16), a partial last N tile and a partial
    last M tile; the columns beyond 448 are not written."""
    M, Kin, Nout, ncol = 1000, 512, 256, 448
    g = torch.Generator(device="cuda").manual_seed(448 + dact)
    dZ = torch.randn(M, Nout, device="cuda", generator=g)
    Wt = (0.1 * torch.randn(Kin, Nout, device="cuda", generator=g)).contiguous()   # W^T [Kin][Nout]
    Y = torch.randn(M, Kin, device="cuda", generator=g) if dact else None
    dX = _gemm_tc(dZ, Nout, 1, Wt, Nout, 1, M, ncol, Nout, Kin, dact=Y, ldd=Kin if dact else 0, dact_n=ncol if dact else 0)
    ref = dZ.double() @ Wt[:ncol].double().t()
    if dact:
        ref = ref * torch.where(Y[:, :ncol] > 0, 1.0, 0.01).double()
    assert _rel(dX[:, :ncol], ref) < 2e-5
    assert torch.all(dX[:, ncol:] == 7.0)


@pytest.mark.parametrize("rows,Kin,Nout,splits", [(5000, 288, 256, 3), (130000, 256, 256, 64), (999, 128, 128, 2), (40000, 272, 256, 20),
                                                  # F = 63 block1.0 dW (Kin 512) at the backward's split counts: the 2-split
                                                  # clamp, (rows + 2047) / 2048, and the 64-split cap
                                                  (3000, 512, 256, 2), (40000, 512, 256, 20), (130000, 512, 256, 64)] +
                         # the reduction rows of a small batch at gemm_tn_acc's split count: 1..32 rows run one split (kchunk 32)
                         # through the workspace, 33 leaves the second split one row, and either side of the 2048-row slabs
                         [(r, kin, nout, grad_check.dw_splits(r)[0]) for r, kin, nout in (
                             (1, 288, 128), (2, 128, 128), (31, 256, 256), (32, 272, 256), (33, 512, 256), (2047, 256, 256),
                             (2048, 288, 128), (2049, 272, 256), (4097, 512, 256))])
def test_gemm_tc_tn_splitk_accumulate(rows, Kin, Nout, splits):
    """dWt[Kin x Nout] += X^T dZ: both operands transposed on the way into shared memory, deterministic split-K, accumulation."""
    assert splits == grad_check.dw_splits(rows)[0], "not the split count the backward passes"
    print("\n[gemm_tc tn] rows=%d Kin=%d Nout=%d splits (asked, run) %s" % (rows, Kin, Nout, grad_check.dw_splits(rows)))
    g = torch.Generator(device="cuda").manual_seed(rows)
    X = torch.randn(rows, Kin, device="cuda", generator=g)
    dZ = torch.randn(rows, Nout + 16, device="cuda", generator=g)[:, :Nout]
    C0 = torch.randn(Kin, Nout, device="cuda", generator=g)
    out = _gemm_tc(X, 1, Kin, dZ, 1, dZ.stride(0), Kin, Nout, rows, Nout, splits=splits, C0=C0)
    ref = C0.double() + X.double().t() @ dZ.double()
    assert _rel(out, ref) < 2e-5
    assert _rel(out.double() - C0.double(), ref - C0.double()) < 2e-5                # the product alone: not hidden by C0's scale
    out2 = _gemm_tc(X, 1, Kin, dZ, 1, dZ.stride(0), Kin, Nout, rows, Nout, splits=splits, C0=C0)
    assert torch.equal(out, out2)                                                   # deterministic (no atomics)
