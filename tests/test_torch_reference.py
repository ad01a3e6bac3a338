"""CPU checks of the float64 modes of oracle/torch_backbone.run_graph that the per-kernel GPU tests rely on: the TF32 rounding, the
magnitude pass, starting buffer contents, and where the rounding is applied."""
import numpy as np
import torch

from hyperpose_b200 import models
from oracle import torch_backbone


def test_tf32_round_is_nearest_ties_away():
    one = 1.0
    ulp = 2.0 ** -10
    x = torch.tensor([one + ulp / 2, -(one + ulp / 2), one + ulp / 2 - 2.0 ** -20, one + 1.5 * ulp, torch.finfo(torch.float32).max, float("inf"), 0.0],
                     dtype=torch.float32)
    want = [one + ulp, -(one + ulp), one, one + 2 * ulp, float("inf"), float("inf"), 0.0]
    assert torch_backbone.tf32_round(x).tolist() == want
    assert torch_backbone.tf32_round(x.double()).dtype == torch.float64


def _one_conv(rng, cin=8, cout=8, res_mode=0):
    g = models.Graph("t", out_down_shift=0)
    a = g.add_buffer(cin, 0); b = g.add_buffer(cout, 0); r = g.add_buffer(cout, 0)
    w = rng.standard_normal((1, cout, cin, 3, 3)).astype(np.float32)
    g.add_conv(a, b, w, rng.standard_normal(cout).astype(np.float32), rng.uniform(-0.5, 1, cout).astype(np.float32),
               res_buf=r, res_mode=res_mode)
    return g, w


def test_float64_modes_of_run_graph():
    rng = np.random.default_rng(0)
    g, w = _one_conv(rng, res_mode=2)
    N, H, W = 2, 5, 6
    x = rng.standard_normal((N, 8, H, W))
    res = rng.standard_normal((N, 8, H, W))
    frames = np.zeros((N, H, W, 3), np.uint8)
    kw = dict(device="cpu", dtype=torch.float64, init={0: x, 2: res}, rounding="fp16")
    _, _, exact = torch_backbone.run_graph(g, frames, round_stores=False, **kw)
    _, _, stored = torch_backbone.run_graph(g, frames, **kw)
    _, _, mag = torch_backbone.run_graph(g, frames, round_stores=False, magnitude=True, **kw)
    out = exact[1].numpy()
    assert exact[1].dtype == torch.float64
    # stores are rounded onto the fp16 grid, and only there; the inputs the test wrote stay as given
    assert np.array_equal(stored[1].numpy(), out.astype(np.float16).astype(np.float64))
    assert not np.array_equal(out, out.astype(np.float16).astype(np.float64))
    assert np.array_equal(exact[0].numpy(), x) and np.array_equal(exact[2].numpy(), res)
    # the weights are rounded onto the grid: a plain float64 conv with fp16 weights gives the same output
    wq = torch.from_numpy(w[0].astype(np.float16).astype(np.float64))
    op = g.ops[0]
    y = torch.nn.functional.conv2d(torch.from_numpy(x), wq, torch.from_numpy(op.bias.astype(np.float64)), padding=1)
    y = torch.where(y > 0, y, y * torch.from_numpy(op.alpha.astype(np.float64)).view(1, -1, 1, 1)) + torch.from_numpy(res)
    assert np.allclose(out, y.numpy(), rtol=0, atol=1e-12)
    # magnitude pass: sum |w x| + |b| + |res| for every output
    m = torch.nn.functional.conv2d(torch.from_numpy(np.abs(x)), wq.abs(), torch.from_numpy(np.abs(op.bias).astype(np.float64)), padding=1)
    assert np.allclose(mag[1].numpy(), (m + torch.from_numpy(np.abs(res))).numpy(), rtol=0, atol=1e-12)
    assert (mag[1].numpy() >= np.abs(out) - 1e-12).all()
