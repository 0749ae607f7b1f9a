"""GPU: the engine's GEMM dispatch (CUDA-core skinny kernel and bf16 tensor-core kernel) against a plain
torch fp32 matmul of the same operands."""
import pytest
import torch

from util import test_gemm as run_gemm

pytestmark = pytest.mark.gpu

SHAPES = [  # (M, N, K)
    (2, 3072, 1024), (2, 1024, 2816), (8, 2304, 768), (5, 16384, 1024),          # skinny (batch-1 latency path)
    (16, 3072, 1024), (33, 1024, 1024), (64, 5632, 1024), (128, 1024, 2816),     # tensor-core path, split-K
    (128, 16384, 1024), (130, 2048, 768), (256, 3072, 1024), (1920, 1280, 2048),  # multi-tile M (t2i prefill)
    (32, 9600, 3200), (24, 3200, 8704),                                           # GPT-3B shapes (K=50*64, 136*64)
]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("path", ["mma", "tcgen05"])
def test_gemm_bf16(M, N, K, path, monkeypatch):
    """path=tcgen05 (test id kept stable; the kernel is wgmma + TMA) routes 8 < M <= 256 through gemm_tc.cu; other shapes fall back."""
    monkeypatch.setenv("LG_GEMM_TC", "1" if path == "tcgen05" else "0")
    torch.manual_seed(M * 7 + N + K)
    x = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    y = run_gemm(x, w)
    ref = x.float() @ w.float().t()
    err = (y - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), err      # fp32 accumulate: reduction-order noise only


@pytest.mark.parametrize("M,N,K", [(2, 3072, 1024), (9, 1024, 2816), (20, 2048, 768), (3, 512, 4096)])
def test_gemm_fp32_exact_mode(M, N, K):
    torch.manual_seed(N)
    x = torch.randn(M, K, device="cuda") * 0.5
    w = torch.randn(N, K, device="cuda") * 0.05
    y = run_gemm(x, w)
    ref = (x.double() @ w.double().t()).float()
    assert (y - ref).abs().max().item() <= 1e-4

