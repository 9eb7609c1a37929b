"""wgmma fused Linear+bias+ReLU vs a plain PyTorch fp32 reference of the same op."""
import pytest
import torch

from eventgrad_b200.ops.linear_tc import linear_act, linear_tc_forward, tc_eligible

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,K,N", [(128, 64, 128), (1000, 784, 128), (300, 128, 256), (77, 16, 16), (4096, 784, 64),
                                   (129, 200, 32), (60000, 784, 128)])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("out", [torch.bfloat16, torch.float32])
def test_linear_tc_forward(M, K, N, relu, out):
    g = torch.Generator(device="cuda").manual_seed(M + K + N)
    x = torch.randn(M, K, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).to(torch.bfloat16)
    b = torch.randn(N, generator=g, device="cuda")
    assert tc_eligible(x, w)
    y = linear_tc_forward(x, w, b, relu, out)
    ref = x.float() @ w.float().t() + b
    if relu:
        ref = ref.relu()
    tol = 2e-2 if out == torch.bfloat16 else 2e-3
    torch.testing.assert_close(y.float(), ref, rtol=tol, atol=tol)


def test_linear_tc_autograd_matches_torch():
    x = torch.randn(512, 784, device="cuda").to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(128, 784, device="cuda") * 0.03).to(torch.bfloat16).requires_grad_(True)
    b = torch.randn(128, device="cuda", requires_grad=True)
    dy = torch.randn(512, 128, device="cuda").to(torch.bfloat16)
    y = linear_act(x, w, b, relu=True)
    y.backward(dy)
    xr, wr, br = [t.detach().float().requires_grad_(True) for t in (x, w, b)]
    yr = (xr @ wr.t() + br).relu()
    yr.backward(dy.float())
    torch.testing.assert_close(y.float(), yr, rtol=2e-2, atol=2e-2)
    for a, r in ((x.grad, xr.grad), (w.grad, wr.grad), (b.grad, br.grad)):
        assert float((a.float() - r).norm() / (r.norm() + 1e-9)) < 2e-2


def test_mlp_uses_tc_path_under_autocast():
    from eventgrad_b200.models import build_model
    torch.manual_seed(0)
    m = build_model("mlp").cuda()
    x = torch.randn(256, 1, 28, 28, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = m(x)
    ref = m(x)          # fp32 path
    torch.testing.assert_close(y.float(), ref, rtol=5e-2, atol=5e-2)
