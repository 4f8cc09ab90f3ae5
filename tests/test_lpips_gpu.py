"""LPIPS (VGG) on the GPU (-m gpu, DESIGN.md section 4.15): the reference's fp32 and fp64 values on the golden cases
(tests/golden/lpips.npz), the fp64 restatement at evaluation and full-HD sizes, each conv layer against F.conv2d in
fp64, max pooling and the head's epsilon exactly, determinism across runs, batch sizes and batch contents, and the
metrics CLI's --lpips_weights end to end."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import instantsplat_b200 as I
from instantsplat_b200 import lpips as LP
from instantsplat_b200 import metrics as M
from oracle.lpips_oracle import lpips_vgg_fp64, seeded_weights, weights_of

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "lpips.npz")


def bound(ref):
    return 1e-7 + 1e-4 * abs(ref)


@pytest.fixture(scope="module")
def weights():
    z = np.load(GOLD)
    vgg, lin, sha = seeded_weights(int(z["seed"]))
    assert sha == str(z["sha256"])
    return vgg, lin


@pytest.fixture(scope="module")
def net(weights):
    return LP.LpipsVGG(*LP.check_weights(*weights), device=DEV)


def _f(u8):
    return torch.from_numpy(np.ascontiguousarray(u8)).to(DEV).permute(2, 0, 1)[None].float().div(255).contiguous()


def test_golden_cases_match_reference(net):
    z = np.load(GOLD)
    worst = 0.0
    for name in z["cases"].tolist():
        got, layers = net(_f(z[f"x_{name}"]), _f(z[f"y_{name}"]))
        got, layers = float(got[0]), layers[0].cpu().numpy()
        for prec in ("32", "64"):
            ref, ref_l = float(z[f"ref{prec}_{name}"]), z[f"layers{prec}_{name}"]
            assert abs(got - ref) <= bound(ref), (name, prec, got, ref)
            assert np.all(np.abs(layers - ref_l) <= 1e-7 + 1e-4 * np.abs(ref_l)), (name, prec, layers, ref_l)
            worst = max(worst, abs(got - ref) / bound(ref))
        if name == "same":
            assert got == 0.0 and np.all(layers == 0.0)
    print(f"worst |ours - reference| / (1e-7 + 1e-4 |reference|) over the golden cases: {worst:.3g}")


@pytest.mark.parametrize("H,W", [(288, 512), (545, 981), (1080, 1920)])
def test_sizes_match_fp64_restatement(net, weights, H, W):
    g = torch.Generator(device=DEV).manual_seed(H * 7 + W)
    x = torch.rand(1, 3, H, W, device=DEV, generator=g)
    y = (x + 0.05 * torch.randn(1, 3, H, W, device=DEV, generator=g)).clamp(0, 1)
    got, layers = net(x, y)
    with torch.no_grad():
        ref, ref_l = lpips_vgg_fp64(x, y, weights_of(*weights))
    assert abs(float(got[0]) - float(ref[0])) <= bound(float(ref[0])), (float(got[0]), float(ref[0]))
    assert torch.all((layers - ref_l).abs() <= 1e-7 + 1e-4 * ref_l.abs())


def _conv(L, x_nhwc, w, b):
    N, H, W_, cin = x_nhwc.shape
    out = torch.empty(N, H, W_, w.shape[0], device=DEV)
    wp = w.permute(1, 2, 3, 0).contiguous()
    I._lib.check(L.gsb_lpips_conv3x3_relu(N, H, W_, cin, w.shape[0], x_nhwc.data_ptr(), wp.data_ptr(), b.data_ptr(),
                                          out.data_ptr(), I._lib.stream_ptr()), "conv")
    return out


@pytest.mark.parametrize("layer", range(13))
def test_conv_layer_matches_fp64(weights, layer):
    L = I.lib()
    m = LP.VGG_CONV[layer]
    w = weights[0][f"features.{m}.weight"].to(DEV)
    b = weights[0][f"features.{m}.bias"].to(DEV)
    g = torch.Generator(device=DEV).manual_seed(layer)
    for H, W in ((1, 1), (2, 37), (19, 2), (17, 33), (40, 23)):
        x = torch.relu(torch.randn(2, w.shape[1], H, W, device=DEV, generator=g))
        got = _conv(L, x.permute(0, 2, 3, 1).contiguous(), w, b).permute(0, 3, 1, 2)
        ref = torch.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1))
        err = float((got.double() - ref).abs().max())
        assert err <= 1e-5 * float(ref.abs().max()) + 1e-30, (layer, H, W, err)


def test_maxpool_is_exact():
    L = I.lib()
    g = torch.Generator(device=DEV).manual_seed(3)
    for N, H, W, C in ((3, 37, 53, 64), (2, 2, 3, 128), (1, 9, 8, 512), (2, 16, 16, 256)):
        x = torch.randn(N, H, W, C, device=DEV, generator=g)
        out = torch.empty(N, H // 2, W // 2, C, device=DEV)
        I._lib.check(L.gsb_lpips_maxpool2(N, H, W, C, x.data_ptr(), out.data_ptr(), I._lib.stream_ptr()), "pool")
        want = F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
        assert torch.equal(out, want), (N, H, W, C)


def test_head_zero_features_use_the_epsilon():
    """An all-zero feature pixel normalises to 0 (the epsilon is outside the square root), not NaN."""
    L = I.lib()
    V, H, W, C = 2, 5, 7, 64
    g = torch.Generator(device=DEV).manual_seed(9)
    feats = torch.relu(torch.randn(2 * V, H, W, C, device=DEV, generator=g))
    feats[0] = 0.0                          # x of view 0 entirely zero
    feats[V + 1, 2] = 0.0                   # a row of y of view 1
    lin = torch.rand(C, device=DEV, generator=g)
    out = torch.zeros(V, 5, dtype=torch.float64, device=DEV)
    parts = torch.empty(V * 128, dtype=torch.float64, device=DEV)
    I._lib.check(L.gsb_lpips_head(V, H, W, C, feats.data_ptr(), lin.data_ptr(), 2, out.data_ptr(), parts.data_ptr(),
                                  I._lib.stream_ptr()), "head")
    f = feats.double()
    n = f / (f.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    want = ((n[:V] - n[V:]) ** 2 * lin.double()).sum(-1).sum((1, 2))
    assert torch.all(torch.isfinite(out[:, 2]))
    assert torch.allclose(out[:, 2], want, rtol=1e-5, atol=0)
    assert torch.all(out[:, [0, 1, 3, 4]] == 0)


def test_deterministic_across_runs_batches_and_neighbours(net):
    g = torch.Generator(device=DEV).manual_seed(11)
    V, H, W = 12, 45, 70
    x = torch.rand(V, 3, H, W, device=DEV, generator=g)
    y = (x + 0.1 * torch.randn(V, 3, H, W, device=DEV, generator=g)).clamp(0, 1)
    y[4] = x[4]
    a, la = net(x, y, max_batch=12)
    b, lb = net(x, y, max_batch=12)
    assert torch.equal(a, b) and torch.equal(la, lb)
    for mb in (1, 3):
        c, lc = net(x, y, max_batch=mb)
        assert torch.equal(a, c) and torch.equal(la, lc), mb
    one, _ = net(x[5:6], y[5:6])
    assert torch.equal(one, a[5:6])
    assert float(a[4]) == 0.0 and bool(torch.all(a[torch.arange(V) != 4] > 0))


def test_call_does_not_wait_for_the_gpu(net):
    """Every chunk's kernels are queued and the results returned without a synchronising CUDA call."""
    g = torch.Generator(device=DEV).manual_seed(13)
    x = torch.rand(3, 3, 40, 56, device=DEV, generator=g)
    y = torch.rand(3, 3, 40, 56, device=DEV, generator=g)
    want, want_l = net(x, y, max_batch=2)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got, got_l = net(x, y, max_batch=2)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(got, want) and torch.equal(got_l, want_l)


def test_metrics_cli_lpips_end_to_end(tmp_path, weights, net, capsys):
    from test_render_views_gpu import N_TRAIN, ITERS, _source_and_model
    from instantsplat_b200 import render_views as R
    src, model, it = _source_and_model(str(tmp_path))
    base = ["-s", src, "-m", model, "--n_views", str(N_TRAIN), "--iterations", "-1", "-r", "1", "--workers", "2"]
    assert R.main(base + ["--eval", "--optim_test_pose_iter", str(ITERS), "--max_batch", "3"]) == 0
    wdir = tmp_path / "hub"
    wdir.mkdir()
    torch.save(weights[0], wdir / LP.VGG_FILE)
    torch.save(weights[1], wdir / LP.LIN_FILE)
    assert M.main(["-s", src, "-m", model, "--n_views", str(N_TRAIN), "--lpips_weights", str(wdir)]) == 0
    out = capsys.readouterr().out
    method = f"ours_{it}"
    per = json.loads(open(os.path.join(model, "per_view.json")).read())[method]
    res = json.loads(open(os.path.join(model, "results.json")).read())[method]
    assert list(per) == ["SSIM", "PSNR", "LPIPS"] and list(res)[:3] == ["SSIM", "PSNR", "LPIPS"]
    renders, gts, names = M.read_pairs(os.path.join(model, "test", method))
    f = lambda u8: torch.from_numpy(u8).to(DEV).div(255.0).permute(0, 3, 1, 2).contiguous()
    want = net(f(renders), f(gts))[0].cpu()
    assert torch.equal(torch.tensor([per["LPIPS"][n] for n in names], dtype=torch.float64), want)
    assert f"  LPIPS: {res['LPIPS']:>12.7f}" in out.splitlines()
    lines = open(os.path.join(model, "test", method, "metrics.txt")).read().splitlines()
    assert all(ln.endswith(f", LPIPS: {per['LPIPS'][n]:.4f}") for ln, n in zip(lines, names))
