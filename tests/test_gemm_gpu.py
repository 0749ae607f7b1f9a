"""GPU: the engine's GEMM dispatch (CUDA-core skinny kernel and bf16 tensor-core kernel) against a plain
torch fp32 matmul of the same operands."""
import pytest
import torch

from util import gemm_dx
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



# ---------------------------------------------------------------------------------------------- direct-epilogue GEMM (gemm_dx.cu)
DX_SHAPES = [  # (M, N, K): decode rows x output features x reduction
    (64, 1024, 1024), (32, 1024, 1024), (16, 1024, 1024), (128, 1024, 1024),      # GPT-L wo at chain sizes 64/32/16 and unsplit
    (40, 1280, 1280), (7, 1536, 1536), (32, 3200, 3200), (64, 2816, 1024),        # ragged row block, XL / XXL / 3B widths
]


def _rms_ref(x, g, eps):
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (xf * rstd).bfloat16() * g          # norm(x.float()).type_as(x) * weight  (gpt.py:147-148)


@pytest.mark.parametrize("M,N,K", DX_SHAPES)
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("rblk", ["16", "32", "64"])
def test_gemm_dx_plain_and_norm_prologue(M, N, K, norm, rblk, monkeypatch):
    monkeypatch.setenv("LG_DX_RBLK", rblk)
    torch.manual_seed(M + N + K)
    x = (torch.randn(M, K, device="cuda") * 0.7).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    g = (1.0 + 0.2 * torch.randn(K, device="cuda")).bfloat16() if norm else None
    y = gemm_dx(x, w, mode=0, normw=g, eps=1e-5)
    xin = _rms_ref(x, g, 1e-5) if norm else x
    ref = xin.float() @ w.float().t()
    err = (y - ref).abs().max().item()
    # fp32 accumulate; with the norm a value sitting on a bf16 rounding boundary may round the other way (rsqrt vs 1/sqrt)
    assert err <= (6e-3 if norm else 2e-3) * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("M,N,K", [(64, 1024, 1024), (37, 1280, 1280), (128, 1024, 1024)])
def test_gemm_dx_residual_epilogue(M, N, K):
    torch.manual_seed(N + M)
    x = (torch.randn(M, K, device="cuda") * 0.7).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    h0 = torch.randn(M, N, device="cuda").bfloat16()
    h1 = gemm_dx(x, w, mode=1, h=h0)
    y = (x.float() @ w.float().t()).bfloat16()
    ref = (h0.float() + y.float()).bfloat16()                     # h = x + f(x), both bf16 tensors (gpt.py:255)
    d = (h1.float() - ref.float()).abs()
    assert d.max().item() <= 2.0 ** -6 * max(1.0, ref.float().abs().max().item())      # at most one bf16 ulp
    assert (d > 0).float().mean().item() < 0.02


@pytest.mark.parametrize("M,F,K", [(64, 2816, 1024), (32, 2816, 1024), (20, 3584, 1280), (128, 2816, 1024)])
def test_gemm_dx_norm_swiglu(M, F, K):
    torch.manual_seed(F + M)
    x = (torch.randn(M, K, device="cuda") * 0.7).bfloat16()
    w1 = (torch.randn(F, K, device="cuda") * 0.05).bfloat16()
    w3 = (torch.randn(F, K, device="cuda") * 0.05).bfloat16()
    g = (1.0 + 0.2 * torch.randn(K, device="cuda")).bfloat16()
    ff = gemm_dx(x, w1, w3, mode=2, normw=g, eps=1e-5)
    xn = _rms_ref(x, g, 1e-5)
    a = (xn.float() @ w1.float().t()).bfloat16()
    b = (xn.float() @ w3.float().t()).bfloat16()
    ref = torch.nn.functional.silu(a) * b                         # gpt.py:167, bf16 tensors
    d = (ff.float() - ref.float()).abs()
    scale = max(1.0, ref.float().abs().max().item())
    assert d.max().item() <= 0.03 * scale, d.max().item()
    assert d.mean().item() <= 2e-3 * scale, d.mean().item()
