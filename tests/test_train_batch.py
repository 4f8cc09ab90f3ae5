"""Several views per optimizer step on one GPU (-m gpu, DESIGN.md section 4.10): gsb_backward_batch and the batched
loss against V single-view calls added in view order, JointTrainer.step_batch against a restatement from the trainer's
public pieces, step_batch([v]) against step(v), graph replay, binning overflow, checkpoints and refusals -- all bit for
bit (torch.equal)."""
import math

import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import GsbError
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.trainer import SEGMENTS

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _with_big_gaussian(sc):
    """Append one faint Gaussian that covers the whole frame of every view, so k_big_rects has work."""
    p = dict(sc.params)
    one = lambda k, v: torch.cat([p[k], v])
    p["xyz"] = one("xyz", sc.params["xyz"].mean(0, keepdim=True))
    p["rotation"] = one("rotation", torch.tensor([[1.0, 0, 0, 0]]))
    p["scaling"] = one("scaling", torch.full((1, 3), math.log(4.0)))
    p["opacity"] = one("opacity", torch.full((1, 1), -3.0))
    p["f_dc"] = one("f_dc", torch.full((1, 1, 3), 0.3))
    p["f_rest"] = one("f_rest", torch.zeros(1, *p["f_rest"].shape[1:]))
    sc.params = p
    if sc.per_point_lr is not None:
        sc.per_point_lr = torch.cat([sc.per_point_lr.reshape(-1), torch.ones(1)])
    return sc


def _targets(sc, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(sc.n_views, 3, sc.height, sc.width, generator=g).to(DEV)


def _trainer(sc, gts, mip=False, deg=None, use_graph=False, **cfg_kw):
    cfg = I.OptimConfig()
    cfg.mip_kernel_size = 0.1 if mip else None
    for k, v in cfg_kw.items():
        setattr(cfg, k, v)
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg, use_graph=use_graph)
    if deg is not None:
        tr.active_sh_degree = deg
    return tr


def _single(tr, views, gts):
    """V single-view forwards + loss_and_backward, gradients added in view order with torch."""
    acc, rows, sums = None, [], []
    for k, v in enumerate(views):
        tr.render(v)
        tr.loss_and_backward(v, gts[k])
        acc = tr.grads.clone() if acc is None else acc + tr.grads
        rows.append(tr.pose_grad[v].clone())
        sums.append(tr.sums.clone())
    return acc, torch.stack(rows), torch.stack(sums)


def _batched(tr, views, gts):
    """The batched forward, loss and gsb_backward_batch (Frame.backward_batch) of step_batch, without the update."""
    V = len(views)
    b = tr._batch_scratch(V)
    b.sel.copy_(torch.tensor([list(views), list(range(V))]))
    tr._settled(lambda: tr._enqueue_batch(b, gts, False), batch=b)
    others = [v for v in range(tr.n_views) if v not in views]
    assert not tr.pose_grad[others].any()
    return tr.grads.clone(), tr.pose_grad[list(views)].clone(), b.sums.clone()


def _assert_grads_equal(tr, views, gts):
    a, b = _single(tr, views, gts), _batched(tr, views, gts)
    for name, _ in SEGMENTS:
        assert torch.equal(tr.view(a[0], name), tr.view(b[0], name)), name
    assert torch.equal(a[0], b[0])
    assert torch.equal(a[1], b[1]), (a[1], b[1])
    assert torch.equal(a[2], b[2]), (a[2], b[2])
    assert a[0].abs().sum() > 0
    return b


GRAD_CASES = [  # (V, SH degree, mip, blind view position, big Gaussian)
    (1, 3, False, None, False),
    (2, 3, False, None, True),
    (3, 3, False, 1, True),
    (5, 3, False, 4, True),
    (3, 0, False, None, True),
    (3, 3, True, 0, True),
    (5, 0, True, 2, False),
]


@pytest.mark.parametrize("V,deg,mip,blind,big", GRAD_CASES)
def test_backward_batch_equals_single_views(V, deg, mip, blind, big):
    sc = surface_scene(6000, 5, 215, 167, seed=61, sh_degree=3)      # W, H not multiples of 16
    if big:
        sc = _with_big_gaussian(sc)
    gts = _targets(sc, V)
    tr = _trainer(sc, gts, mip=mip, deg=deg)
    views = [4, 1, 3, 0, 2][:V]                                     # not in index order
    if blind is not None:
        tr.poses[views[blind], 4:] = torch.tensor([0.0, 0.0, -100.0], device=DEV)   # sees nothing
    _assert_grads_equal(tr, views, gts[views])
    if big:
        assert int(tr._batch.frame.radii[:, -1].max()) > 215


def test_backward_batch_long_tile_lists():
    """Tile lists in every size class of the per-tile sort, in every view of the batch."""
    from test_binning_lists import lengths_scene
    sc, _ = lengths_scene()
    sc.poses = sc.poses.expand(3, 7).clone()
    gts = _targets(sc, 5)
    tr = _trainer(sc, gts)
    _assert_grads_equal(tr, [2, 0, 1], gts[[2, 0, 1]])
    st = tr._batch.frame.status.cpu().tolist()
    assert st[4] >= 3 and st[5] >= 3, st                          # both long-list queues are non-empty


def test_backward_batch_beyond_65536_tiles():
    sc = surface_scene(3000, 12, 1920, 1080, seed=9, sh_degree=3)
    assert 12 * 120 * 68 > 65536
    gts = _targets(sc, 9)
    tr = _trainer(sc, gts)
    views = list(range(11, -1, -1))
    _assert_grads_equal(tr, views, gts[views])


# ---- training steps --------------------------------------------------------------------------------------------------
def snapshot(tr):
    s = {f"{b}_{k}": tr.view(getattr(tr, b), k).clone() for b in ("params", "exp_avg", "exp_avg_sq") for k, _ in SEGMENTS}
    s.update(poses=tr.poses.clone(), pose_m=tr.pose_m.clone(), pose_v=tr.pose_v.clone(), opt_step=tr.opt_step,
             iteration=tr.iteration, active_sh_degree=tr.active_sh_degree,
             filter_3D=None if tr.filter_3D is None else tr.filter_3D.clone(), mip=list(tr.mip_recomputed_at))
    return s


def assert_same(a, b, where=""):
    assert a.keys() == b.keys()
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), (where, k)
        else:
            assert a[k] == b[k], (where, k, a[k], b[k])


def restated_step(tr, views):
    """One step over `views` from the trainer's public pieces: per view forward + loss_and_backward, gradients summed
    in view order, iteration += V with the schedules' crossings, optimizer_step(grad_scale=1/V)."""
    c, V = tr.cfg, len(views)
    before = tr.iteration
    tr.iteration += V
    if tr.iteration // c.sh_increase_interval > before // c.sh_increase_interval:
        tr.active_sh_degree = min(tr.active_sh_degree + 1, c.max_sh_degree)
    acc, pg, losses = None, None, []
    for v in views:
        tr.render(v)
        tr.loss_and_backward(v, tr.gt[v])
        acc = tr.grads.clone() if acc is None else acc + tr.grads
        pg = tr.pose_grad.clone() if pg is None else pg + tr.pose_grad
        losses.append(tr.loss_value().clone())
    tr.grads.copy_(acc)
    tr.pose_grad.copy_(pg)
    if tr.iteration < c.iterations:
        tr.optimizer_step(grad_scale=1.0 / V)
    if tr.filt is not None and tr.iteration // c.mip_filter3d_interval > before // c.mip_filter3d_interval and \
            tr.iteration < c.iterations - 100:
        tr.compute_filter_3D()
        tr.mip_recomputed_at.append(tr.iteration)
    return torch.stack(losses)


BATCHES = [[0, 1, 2], [3, 4, 0], [2, 4, 1], [1, 0, 3], [4, 2, 3], [0, 2, 4], [3, 1, 0], [2, 3, 4]]


def _scene():
    sc = surface_scene(8000, 5, 120, 88, seed=17, sh_degree=3)
    return sc, _targets(sc, 3)


@pytest.mark.parametrize("use_graph", [False, True])
def test_step_batch_equals_restatement(use_graph):
    sc, gts = _scene()
    kw = dict(mip=True, deg=0, sh_increase_interval=4, mip_filter3d_interval=5)
    a = _trainer(sc, gts, use_graph=use_graph, **kw)
    b = _trainer(sc, gts, **kw)
    for k, views in enumerate(BATCHES):
        a.step_batch(views)
        losses = restated_step(b, views)
        assert_same(snapshot(a), snapshot(b), k)
        assert torch.equal(a.batch_loss_values(), losses), (k, a.batch_loss_values(), losses)
    assert a.active_sh_degree == 3 and len(a.mip_recomputed_at) >= 3
    if use_graph:
        assert any(k[0] == "batch" for k in a._graphs)


@pytest.mark.parametrize("use_graph", [False, True])
def test_step_batch_of_one_view_equals_step(use_graph):
    sc, gts = _scene()
    kw = dict(deg=0, sh_increase_interval=5)
    a = _trainer(sc, gts, use_graph=use_graph, **kw)
    b = _trainer(sc, gts, use_graph=use_graph, **kw)
    for k in range(12):
        v = (3 * k) % 5
        a.step_batch([v])
        b.step(v)
        assert_same(snapshot(a), snapshot(b), k)
        assert torch.equal(a.batch_loss_values()[0], b.loss_value())
        assert torch.equal(a.grads, b.grads) and torch.equal(a.pose_grad, b.pose_grad)


def test_one_graph_serves_every_choice_of_views():
    sc, gts = _scene()
    a = _trainer(sc, gts, use_graph=True)
    b = _trainer(sc, gts)
    a.headroom = b.headroom = 4.0                      # no capacity change, so the graph key stays the same
    for k, views in enumerate(BATCHES):
        a.step_batch(views)
        b.step_batch(views)
        assert_same(snapshot(a), snapshot(b), k)
    keys = [k for k in a._graphs if k[0] == "batch"]
    assert len(keys) == 1, keys
    # explicit targets: another buffer is another key, and one graph again serves every subset
    for views in BATCHES[:3]:
        a.step_batch(views, gts[views].contiguous())
        b.step_batch(views, gts[views].contiguous())
    assert_same(snapshot(a), snapshot(b))


@pytest.mark.parametrize("use_graph", [False, True])
def test_binning_overflow_is_repaired(use_graph):
    """An undersized batch buffer: the step is taken once, with the results of a run that never overflowed.  With
    graph replay the overflow is seen through the batch's own pinned status words, and the repeat replays a graph
    captured at the grown capacity."""
    sc, gts = _scene()
    a, b = _trainer(sc, gts, use_graph=use_graph), _trainer(sc, gts)
    for views in BATCHES[:2]:
        a.step_batch(views)
        b.step_batch(views)
    a._batch.frame.alloc_binning(2000)                 # far below the batch's instance count
    n, steps = a.overflows, a.opt_step
    a.step_batch(BATCHES[2])
    b.step_batch(BATCHES[2])
    assert a.overflows == n + 1 and a.opt_step == steps + 1
    assert a._batch.frame.cap > 2000
    assert_same(snapshot(a), snapshot(b))
    for views in BATCHES[3:5]:
        a.step_batch(views)
        b.step_batch(views)
        assert_same(snapshot(a), snapshot(b))
    assert a.overflows == n + 1


# step() and step_batch() on one trainer.  Each frame numbers its own forwards, so the two counts meet (below, each
# frame's forward 3 follows the other's), with a binning capacity between the two frames' instance counts: a status
# word taken from the other frame would miss a real overflow (batch) or report a false one (single view).  Whether a
# replayed forward's own words have landed before the host first polls depends on timing, so the tests check the
# results against eager runs and, directly, that the two frames copy their words to different pinned slots.
def _both(pair, fn):
    for tr in pair:
        fn(tr)


def _check(pair, where):
    a, b = pair
    assert_same(snapshot(a), snapshot(b), where)
    assert a.overflows == b.overflows, (where, a.overflows, b.overflows)


def _call(call):
    return (lambda t: t.step_batch(call)) if isinstance(call, list) else (lambda t: t.step(call))


@pytest.mark.parametrize("use_graph", [False, True])
def test_step_and_step_batch_interleaved(use_graph):
    """step() and step_batch() interleaved on one trainer, replayed from graphs already captured, give the results of
    the same calls launched eagerly, and each call sees its own frame's instance count."""
    sc, gts = _scene()
    kw = dict(deg=0, sh_increase_interval=6)
    # 1. step_batch is its frame's forward 3 right after step() was the single-view frame's forward 3, and the batch
    #    overflows its capacity (the Gaussians grew) while the single view's last count is below it
    pair = (_trainer(sc, gts, use_graph=use_graph, **kw), _trainer(sc, gts, **kw))
    _both(pair, _call(0))
    _both(pair, _call([1, 2, 3]))
    r_batch = pair[1].last_R
    _both(pair, lambda t: t._batch.frame.alloc_binning(int(1.2 * r_batch)))
    for call in ([2, 4, 0], 4, 1):
        _both(pair, _call(call))
        _check(pair, call)
    assert pair[1].last_R < int(1.2 * r_batch)
    _both(pair, lambda t: t.view(t.params, "scaling").add_(math.log(1.6)))
    n = pair[1].overflows
    _both(pair, _call([3, 0, 1]))
    assert pair[1].overflows == n + 1
    _check(pair, "batch overflow after step")
    for call in ([0, 1, 4], 2):
        _both(pair, _call(call))
        _check(pair, call)
    # 2. step() is its frame's forward 3 right after step_batch was the batch frame's forward 3, and the single view
    #    fits its capacity while the batch's count does not
    pair = (_trainer(sc, gts, use_graph=use_graph, **kw), _trainer(sc, gts, **kw))
    _both(pair, _call(0))
    r_single = pair[1].last_R
    _both(pair, _call([1, 2, 3]))
    r_batch = pair[1].last_R
    assert r_single < r_batch // 2, (r_single, r_batch)
    _both(pair, lambda t: t.frame.alloc_binning((r_single + r_batch) // 2))
    for call in (1, [2, 0, 4], [4, 3, 1]):
        _both(pair, _call(call))
        _check(pair, call)
    n = pair[1].overflows
    _both(pair, _call(3))
    assert pair[1].overflows == n                      # the single view fits
    _check(pair, "step after batches")
    if use_graph:
        assert any(k[0] == "batch" for k in pair[0]._graphs) and any(k[0] != "batch" for k in pair[0]._graphs)
    # each frame's status words travel to their own pinned slot: a poll never sees the other frame's serial number
    a = pair[0]
    assert a._batch.host_status.data_ptr() != a.host_status.data_ptr()
    assert a._batch.host_status.is_pinned()


def test_checkpoint_resume_with_batched_steps(tmp_path):
    sc, gts = _scene()
    kw = dict(deg=0, sh_increase_interval=4)
    full = _trainer(sc, gts, **kw)
    for views in BATCHES:
        full.step_batch(views)
    a = _trainer(sc, gts, **kw)
    for views in BATCHES[:3]:
        a.step_batch(views)
    path = str(tmp_path / "chkpnt.pth")
    a.save_checkpoint(path)
    c = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, device=DEV)
    assert c.iteration == 9 and c.opt_step == 3
    for views in BATCHES[3:]:
        c.step_batch(views)
    assert_same(snapshot(full), snapshot(c))


def test_refusals():
    sc, gts = _scene()
    tr = _trainer(sc, gts)
    for views in ([], [0, 0], [5], [-1]):
        with pytest.raises(ValueError):
            tr.step_batch(views)
    for bad in (gts[:3], gts[[0, 1]].double(), gts[[0, 1]].cpu(), gts[[0, 1], :, :80]):
        with pytest.raises(ValueError):
            tr.step_batch([0, 1], bad)
    with pytest.raises(GsbError):
        tr.batch_loss_values()                         # no step_batch yet
    no_gt = I.JointTrainer(sc, DEV)
    with pytest.raises(ValueError):
        no_gt.step_batch([0])
    d = _trainer(sc, gts, densify=True)
    with pytest.raises(GsbError):
        d.step_batch([0, 1])
    two = I.JointTrainer(sc, DEV, gt_images=gts, world_size=2, rank=0)
    with pytest.raises(GsbError):
        two.step_batch([0, 1])
    assert tr.iteration == 0 and tr.opt_step == 0
