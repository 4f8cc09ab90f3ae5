"""Evaluation metrics on the GPU (-m gpu, DESIGN.md section 4.11): gsb_image_metrics_batch against the reference's own
ssim / l1_loss / psnr (tests/golden/metrics.npz) in both conventions, save_image's 8-bit round trip exactly,
determinism, JointTrainer.evaluate against the training render, evaluate leaving training untouched, and
PoseTracker.evaluate_batch against render_batch."""
import os

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import GsbError
from instantsplat_b200.evaluation import image_metrics
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.trainer import SEGMENTS
from instantsplat_b200.tracking import PoseTracker
from test_train_batch import _targets, _trainer, assert_same, snapshot

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz")


def _equal(a, b, where=""):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), (where, k, a[k], b[k])


def _rows(m, idx):
    return {k: v[idx] for k, v in m.items()}


@pytest.mark.parametrize("name", ["small", "big"])
@pytest.mark.parametrize("mode", ["clamp", "png8"])
def test_against_reference_golden(name, mode):
    z = np.load(GOLD)
    r, g = torch.from_numpy(z[f"{name}_render"]).to(DEV), torch.from_numpy(z[f"{name}_gt"]).to(DEV)
    m = {k: v.cpu().numpy() for k, v in image_metrics(r, g, mode=mode).items()}
    l1 = z[f"{name}_{mode}_l1"]
    assert np.all(np.abs(m["l1"] - l1) <= 1e-6 * l1), (m["l1"], l1)
    assert np.all(np.abs(m["ssim"] - z[f"{name}_{mode}_ssim"]) <= 2e-6), (m["ssim"], z[f"{name}_{mode}_ssim"])
    for key in ("psnr", "psnr_channels"):
        got, want = m[key], z[f"{name}_{mode}_{key}"]
        assert np.array_equal(np.isinf(got), np.isinf(want)), (key, got, want)
        fin = np.isfinite(want)
        assert np.all(np.abs(got[fin] - want[fin]) <= 1e-4), (key, got, want)


def test_png8_quantisation_is_exact():
    """Tie values (x * 255 == k + 0.5 in fp32) and their neighbours, one per 32x16 tile against a zero target: every
    partial is one value, so the fp64 sums are exact, and sum |a - b| must be torchvision's to 1e-12.  Rounding ties
    to even moves a whole level; multiplying by 1/255 moves 126 levels by one ulp (about 1e-11 of this sum)."""
    z = np.load(GOLD)
    ties, want = z["ties"], z["ties_png8"]
    vals = torch.zeros(3 * 16 * 16)
    vals[:len(ties)] = torch.from_numpy(ties)
    img = torch.zeros(1, 3, 16 * 16, 32 * 16)
    img.view(3, 16, 16, 16, 32)[:, :, 0, :, 0] = vals.view(3, 16, 16)
    assert int((img != 0).sum()) == int((vals != 0).sum())
    m = image_metrics(img.to(DEV), torch.zeros_like(img, device=DEV), mode="png8")
    n = 3 * img.shape[2] * img.shape[3]
    got = float(m["l1"][0]) * n
    exp = float(np.sum(want.astype(np.float64)))
    assert abs(got - exp) <= 1e-12 * exp, (got, exp, got - exp)


def _random_views(V, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    imgs = torch.rand(V, 3, H, W, generator=g) * 1.2 - 0.1
    gts = (imgs + 0.15 * torch.randn(V, 3, H, W, generator=g)).float()
    return imgs.to(DEV), gts.to(DEV)


@pytest.mark.parametrize("mode", ["clamp", "png8"])
def test_deterministic_and_independent_of_the_batch(mode):
    V = 5
    imgs, gts = _random_views(V, 270, 481, 11)
    full = image_metrics(imgs, gts, mode=mode)
    _equal(full, image_metrics(imgs, gts, mode=mode), "repeat")
    rev = list(range(V))[::-1]
    _equal(_rows(full, rev), image_metrics(imgs.flip(0).contiguous(), gts, rows=rev, mode=mode), "reversed")
    for v in range(V):
        alone = image_metrics(imgs[v:v + 1], gts, rows=[v], mode=mode)
        _equal(_rows(full, [v]), alone, v)
        # first and last of a batch with other views
        others = [u for u in range(V) if u != v]
        first = image_metrics(torch.cat([imgs[v:v + 1], imgs[others]]), gts, rows=[v] + others, mode=mode)
        last = image_metrics(torch.cat([imgs[others], imgs[v:v + 1]]), gts, rows=others + [v], mode=mode)
        _equal(_rows(full, [v]), _rows(first, [0]), ("first", v))
        _equal(_rows(full, [v]), _rows(last, [V - 1]), ("last", v))


def _scene():
    sc = surface_scene(8000, 5, 120, 88, seed=17, sh_degree=3)
    return sc, _targets(sc, 3)


@pytest.mark.parametrize("deg", [1, 3])
@pytest.mark.parametrize("mip", [False, True])
def test_evaluate_matches_training_render(deg, mip):
    sc, gts = _scene()
    tr = _trainer(sc, gts, mip=mip, deg=deg)
    views = [3, 0, 4, 1]
    for mode in ("clamp", "png8"):
        ev = tr.evaluate(views, mode=mode)
        renders = torch.stack([tr.render(v).clone() for v in views])
        _equal(ev, image_metrics(renders, tr.gt, rows=views, mode=mode), mode)
        _equal(ev, tr.evaluate(poses=tr.poses[views].clone(), gts=tr.gt[views].clone(), mode=mode), "poses")
        for b in (1, 2, 3):
            _equal(ev, tr.evaluate(views, mode=mode, max_batch=b), ("max_batch", b))
    allv = tr.evaluate()
    assert allv["psnr"].shape == (sc.n_views,)
    _equal(_rows(allv, views), tr.evaluate(views), "default views")


def _state(tr, loss):
    s = snapshot(tr)
    s.update(loss=loss.clone(), grads=tr.grads.clone(), opt_step=tr.opt_step, lag=dict(tr._lag), P=tr.P,
             densified_at=list(tr.densified_at), reset_at=list(tr.reset_at))
    return s


@pytest.mark.parametrize("how", ["eager", "graph", "batch_densify"])
def test_evaluate_changes_nothing(how):
    sc, gts = _scene()
    kw = dict(deg=0, sh_increase_interval=4)
    if how == "batch_densify":
        kw.update(densify=True, densify_batches=True, densify_from_iter=2, densify_until_iter=100,
                  densification_interval=4, opacity_reset_interval=9, iterations=1000)
    graph = how == "graph"
    a, b = _trainer(sc, gts, use_graph=graph, **kw), _trainer(sc, gts, use_graph=graph, **kw)
    for k in range(8):
        for t in (a, b):
            if how == "batch_densify":
                t.step_batch([k % 5, (k + 2) % 5])
            else:
                t.step(k % 5)
        a.evaluate(mode="clamp" if k % 2 else "png8", max_batch=2 if k % 3 == 0 else None)
        loss = (lambda t: t.batch_loss_values()) if how == "batch_densify" else (lambda t: t.loss_value())
        assert_same(_state(a, loss(a)), _state(b, loss(b)), (how, k))
        assert a.last_R == b.last_R and a.cap == b.cap and a.overflows == b.overflows
    for name, _ in SEGMENTS:
        assert a.step_count(name) == b.step_count(name)
    if graph:
        assert len(a._graphs) == len(b._graphs) > 0
    if how == "batch_densify":
        assert a.densified_at and a.reset_at


def _tracker(sc):
    p = sc.params
    return PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width,
                       sc.height, sc.fovx, sc.fovy, sh_degree=3, device=DEV)


def test_tracker_evaluate_batch():
    sc, gts = _scene()
    tk = _tracker(sc)
    init = sc.poses.to(DEV).clone()
    init[:, 4:] += 0.02
    best, _ = tk.optimize_batch(init, gts, num_iter=4)
    m = tk.evaluate_batch(best, gts)
    _equal(m, image_metrics(tk.render_batch(best), gts, mode="png8"), "render_batch")
    _equal(m, tk.evaluate_batch(best, gts, max_batch=2), "max_batch")
    for v in range(sc.n_views):
        _equal(_rows(m, [v]), tk.evaluate_batch(best[v:v + 1], gts[v:v + 1]), v)
    c = tk.evaluate_batch(best, gts, mode="clamp")
    assert not torch.equal(c["l1"], m["l1"])


def test_refusals():
    sc, gts = _scene()
    tr = _trainer(sc, gts)
    with pytest.raises(ValueError, match="not both"):
        tr.evaluate([0], poses=tr.poses[:1].clone(), gts=gts[:1])
    with pytest.raises(ValueError, match="out of range"):
        tr.evaluate([0, 5])
    with pytest.raises(ValueError, match="out of range"):
        tr.evaluate([-1])
    with pytest.raises(ValueError, match="mode"):
        tr.evaluate(mode="png")
    with pytest.raises(ValueError, match="max_batch"):
        tr.evaluate(max_batch=0)
    with pytest.raises(ValueError, match="shape"):
        tr.evaluate([0, 1], gts=gts[:1])
    with pytest.raises(ValueError, match="float32"):
        tr.evaluate([0], gts=gts[:1].double())
    with pytest.raises(ValueError, match="CUDA"):
        tr.evaluate([0], gts=gts[:1].cpu())
    with pytest.raises(ValueError, match="poses"):
        tr.evaluate(poses=tr.poses[:2, :6].clone(), gts=gts[:2])
    with pytest.raises(ValueError, match="poses"):
        tr.evaluate(poses=tr.poses[:2].cpu(), gts=gts[:2])
    with pytest.raises(ValueError, match="gts"):
        tr.evaluate(poses=tr.poses[:2].clone())
    with pytest.raises(ValueError, match="no views"):
        tr.evaluate([])
    tk = _tracker(sc)
    p = sc.poses.to(DEV)
    with pytest.raises(ValueError, match="gts"):
        tk.evaluate_batch(p, gts[:2])
    with pytest.raises(ValueError, match=r"\[V, 7\]"):
        tk.evaluate_batch(p[:, :6], gts)
    with pytest.raises(ValueError, match="mode"):
        tk.evaluate_batch(p, gts, mode="jpeg")
    with pytest.raises(ValueError, match="max_batch"):
        tk.evaluate_batch(p, gts, max_batch=0)
    x = gts[:2].contiguous()
    with pytest.raises(ValueError, match="out of range"):
        image_metrics(x, x, rows=[0, 2])
    with pytest.raises(ValueError, match="rows"):
        image_metrics(x, x, rows=[0])
    with pytest.raises(ValueError, match="frame size"):
        image_metrics(x, x[:, :, :-1].contiguous())
    # V * C beyond the grid's z limit: refused by the library
    many = torch.zeros(21846, 3, 1, 1, device=DEV)
    with pytest.raises(GsbError, match="invalid argument"):
        image_metrics(many, many)
    L = I.lib()
    out = torch.zeros(1, 5, dtype=torch.float64, device=DEV)
    rows = torch.zeros(1, dtype=torch.int32, device=DEV)
    need = L.gsb_image_metrics_scratch_bytes(1, 3, 88, 120)
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    args = (1, 3, 88, 120, x.data_ptr(), x.data_ptr(), rows.data_ptr())
    assert L.gsb_image_metrics_batch(*args, 3, out.data_ptr(), scratch.data_ptr(), need, 0) == -1
    assert L.gsb_image_metrics_batch(*args, 1, out.data_ptr(), scratch.data_ptr(), need - 8, 0) == -1
    assert L.gsb_image_metrics_batch(*args, 1, out.data_ptr(), scratch.data_ptr(), need, 0) == 0
    torch.cuda.synchronize()
