"""GPU tests of the GEMM epilogues that store through shared memory and TMA (bf16, fp32, +residual, deterministic
split-K partial tiles), for every operand major-ness and both tile widths (N < 256: BN 128; N >= 256: BN 256), against
fp32 torch math.  Every case also checks that the store clips at M and N: pad columns of a pitched C (ldc > N) and the
neighbouring columns of a C that is a column slice of a wider tensor keep their contents."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from open_muse_b200 import _lib, ops  # noqa: E402

DEV = "cuda"
EPI_SPLITK_F32 = 4  # reached through muse_gemm_bf16_splitk (workspace + ordered reduction)
FILL = 7.0


def _rand(shape, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g).to(dtype).to(DEV)


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _gemm(epi, A, B, C, res, M, N, K, ldc, a_mn, b_mn):
    if epi != EPI_SPLITK_F32:
        return ops.gemm(A, B, C, M, N, K, A.stride(0), B.stride(0), ldc, a_mn, b_mn, epi, res=res)
    need = _lib.load().muse_gemm_splitk_workspace_bytes(M, N, K)
    ws = torch.empty(max(need, 16) // 4, dtype=torch.float32, device=DEV)
    ops._call("muse_gemm_bf16_splitk", ops._p(A), ops._p(B), ops._p(C), M, N, K, A.stride(0), B.stride(0), ldc, a_mn,
              b_mn, ops._p(ws), need, ops._prep(C))


@pytest.mark.parametrize("K", [512, 2048])
@pytest.mark.parametrize("N", [72, 200, 320, 1000, 2048])
@pytest.mark.parametrize("majors", [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize("epi", ["bf16", "f32", "resadd", "splitk"])
def test_gemm_epilogue(epi, majors, N, K):
    M = 200  # not a multiple of the 128-row tile
    a_mn, b_mn = majors
    code = {"bf16": ops.EPI_BF16, "f32": ops.EPI_F32, "resadd": ops.EPI_RESADD_F32, "splitk": EPI_SPLITK_F32}[epi]
    dt = torch.bfloat16 if epi == "bf16" else torch.float32
    A = _rand((K, M) if a_mn else (M, K), 11)
    B = _rand((K, N) if b_mn else (N, K), 12)
    ref = (A.float().t() if a_mn else A.float()) @ (B.float() if b_mn else B.float().t())
    tol = {"bf16": 6e-3, "f32": 1e-5, "resadd": 6e-3, "splitk": 1e-5}[epi]
    npad = (N + 7) // 8 * 8
    # (pitch, first column of C): C with pad columns past N, and C as a column slice of a wider tensor
    for width, off in [(npad + 8, 0), (npad + 24, 8)]:
        full = torch.full((M, width), FILL, dtype=dt, device=DEV)
        C = full[:, off:off + N]
        res = None
        if epi == "resadd":
            res_full = torch.randn(M, width, generator=torch.Generator().manual_seed(13)).to(DEV)
            res = res_full[:, off:off + N]
        _gemm(code, A, B, C, res, M, N, K, width, a_mn, b_mn)
        torch.cuda.synchronize()
        if epi == "resadd":
            # the same accumulators as the fp32 epilogue, rounded to bf16 and added to the residual in fp32
            acc = torch.empty(M, N, dtype=torch.float32, device=DEV)
            _gemm(ops.EPI_F32, A, B, acc, None, M, N, K, N, a_mn, b_mn)
            torch.cuda.synchronize()
            assert torch.equal(C, res + acc.to(torch.bfloat16).float()), (width, off)
            assert _rel(C - res, ref) < tol, (width, off)
        else:
            assert _rel(C, ref) < tol, (width, off)
        untouched = torch.cat([full[:, :off], full[:, off + N:]], dim=1)
        assert bool((untouched == FILL).all()), (width, off)
