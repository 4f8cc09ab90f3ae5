"""The optimizer kernels against the restatements of test_optimizer_edges_cpu.py at their edges (-m gpu).

k_adam_gate + k_adam (gs_adam.cu, PerPointAdam and every JointTrainer step): each case is checked against two arms,
the kernel's own arithmetic in numpy float32 (bit for bit; with weight decay, within a bound on the FMA) and the
reference optimizer in float64 on the same fp32 constants (within a few fp32 roundings of the terms), always from the
kernel's previous state so that errors do not compound.  Cases: the whole-tensor gate false on long tensors, opened
by one element at either end, -0.0, weight decay, grad_scale, Inf and NaN elements (a NaN freezes the moments, as
grad.norm() > 0 does in the reference); per-row learning rates at row lengths 1, 3, 7, 45 on the vector and scalar
paths; sizes around the 2048-element block; zero-size tensors in a launch; more than 8 tensors; the skip word and
device-side step sizes; 50 steps of PerPointAdam.
k_fused_rs_adam_ag (gs_comm.cu) on one GPU standing in for W = 2, 3, 8 ranks: bit for bit the single-GPU step on the
rank-order sum of the gradients.  k_track_step (gs_track.cu): torch.optim.Adam in float64 over 500 steps, the best
candidate bookkeeping, and batches equal to single-view launches bit for bit.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from test_optimizer_edges_cpu import F32, F64, U, adam32, adam64, adam_bounds, close_within, consts, same_bits
from instantsplat_b200 import _lib
from instantsplat_b200._lib import GsbAdamTensor, GsbError, GsbShardPiece
from instantsplat_b200.per_point_adam import PerPointAdam, launch_adam
from instantsplat_b200.trainer import flat_layout

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHUNK = 2048                   # elements per k_adam block
SLOTS = 84                     # tensors of 84 k + j chunks: neither a whole number of 84-CTA waves nor of blocks
FLAG_NONZERO, FLAG_NAN = 1, 256


def K():
    return _lib.lib()


class Case:
    """One tensor of an Adam launch: device p, g, m, v (views `offset` floats into their allocations), its
    per-row multiplier and hyper-parameters."""

    def __init__(self, n, seed, grad="rand", row_len=1, ppl=False, offset=0, step=1e-3, gscale=1.0, wd=0.0,
                 eps=1e-15, beta1=0.9, beta2=0.999, gmag=1.0):
        r = np.random.default_rng(seed)
        self.n, self.row_len, self.step = n, row_len, step
        self.hp = dict(beta1=beta1, beta2=beta2, eps=eps, weight_decay=wd, grad_scale=gscale)
        self.c = consts(**self.hp)
        host = lambda a: torch.from_numpy(np.concatenate([np.full(offset, 7.0, F32), a.astype(F32)]))
        g = (r.standard_normal(n) * gmag).astype(F32) if isinstance(grad, str) else np.asarray(grad, F32)
        self._p, self._g = host(r.standard_normal(n)).to(DEV), host(g).to(DEV)
        self._m, self._v = host(r.standard_normal(n) * 0.05).to(DEV), host(r.random(n) * 1e-3).to(DEV)
        self.p, self.g, self.m, self.v = (t[offset:] for t in (self._p, self._g, self._m, self._v))
        self.ppl = None
        if ppl:
            rows = n // row_len
            self.ppl = torch.from_numpy(r.uniform(0.25, 4.0, rows).astype(F32)).to(DEV)
        self._dummy = torch.zeros(4, device=DEV)

    def set_grad(self, g):
        self.g.copy_(torch.as_tensor(np.asarray(g, F32)))

    def abi(self, t, host_step=True):
        ptr = lambda x: x.data_ptr() if self.n else self._dummy.data_ptr()
        t.param, t.grad, t.exp_avg, t.exp_avg_sq = ptr(self.p), ptr(self.g), ptr(self.m), ptr(self.v)
        t.per_point_lr = None if self.ppl is None else self.ppl.data_ptr()
        t.numel, t.row_len = self.n, self.row_len
        t.step_size = self.step if host_step else 0.0
        t.beta1, t.beta2, t.eps = self.hp["beta1"], self.hp["beta2"], self.hp["eps"]
        t.weight_decay, t.grad_scale = self.hp["weight_decay"], self.hp["grad_scale"]

    def entry(self):
        return dict(param=self.p, grad=self.g, exp_avg=self.m, exp_avg_sq=self.v, per_point_lr=self.ppl,
                    step_size=self.step, row_len=self.row_len, **self.hp)

    def snap(self):
        return tuple(t.cpu().numpy().copy() for t in (self.p, self.g, self.m, self.v))

    def lr_mul(self):
        return None if self.ppl is None else np.repeat(self.ppl.cpu().numpy(), self.row_len)


def launch(cases, skip=None, step_dev=None, flags=None):
    arr = (GsbAdamTensor * len(cases))()
    for t, c in zip(arr, cases):
        c.abi(t, host_step=step_dev is None)
    flags = torch.zeros(8, dtype=torch.int32, device=DEV) if flags is None else flags
    rc = K().gsb_adam_step_ex(len(cases), arr, flags.data_ptr(), None if skip is None else skip.data_ptr(),
                              None if step_dev is None else step_dev.data_ptr(), _lib.stream_ptr())
    torch.cuda.synchronize()
    return rc, flags.cpu().numpy()


def expected_flag(g, p, c):
    with np.errstate(all="ignore"):
        gd = (g * c["gscale"]).astype(F32)
        if c["wd"] != 0:
            gd = (gd.astype(F64) + F64(c["wd"]) * p.astype(F64)).astype(F32)
        return (FLAG_NONZERO if np.any(gd * gd > 0) else 0) | (FLAG_NAN if np.any(np.isnan(gd)) else 0)


def check_step(case, before, label=""):
    """Both arms for one case after one step from `before` (p, g, m, v on the host)."""
    p0, g0, m0, v0 = before
    got = case.snap()
    p1, m1, v1 = got[0], got[2], got[3]
    lm = case.lr_mul()
    e32 = adam32(p0, g0, m0, v0, case.step, case.c, lr_mul=lm)
    if case.c["wd"] == 0:
        for name, a, b in zip("pmv", (p1, m1, v1), e32):
            assert same_bits(a, b), f"{label}: {name} differs from the fp32 restatement"
    else:             # the kernel's FMA rounds the decayed gradient once, the restatement may round it twice
        bm, bv, bp = adam_bounds(p0, g0, m0, v0, case.step, case.c, lr_mul=lm)
        for name, a, b, bd in zip("pmv", (p1, m1, v1), e32, (bp, bm, bv)):
            assert close_within(a, b, bd), f"{label}: {name} beyond the FMA bound of the fp32 restatement"
    rows = case.n // case.row_len
    shp = (rows, case.row_len)
    e64 = adam64(p0.reshape(shp), g0.reshape(shp), m0.reshape(shp), v0.reshape(shp), case.step, case.c,
                 ppl=None if case.ppl is None else case.ppl.cpu().numpy().reshape(rows, 1))
    bm, bv, bp = adam_bounds(p0, g0, m0, v0, case.step, case.c, lr_mul=lm)
    for name, a, b, bd in zip("pmv", (p1, m1, v1), e64, (bp, bm, bv)):
        assert close_within(a, b.reshape(-1), bd), f"{label}: {name} beyond the fp64 reference's bound"


def run_and_check(cases, label=""):
    before = [c.snap() for c in cases]
    rc, flags = launch(cases)
    assert rc == 0
    for k, (c, b) in enumerate(zip(cases, before)):
        if c.n:
            assert flags[k] == expected_flag(b[1], b[0], c.c), f"{label}: tensor {k} flag {flags[k]}"
            check_step(c, b, f"{label} tensor {k} (n={c.n})")
    return before


# ---- A. gsb_adam_step_ex / PerPointAdam ---------------------------------------------------------------------------
def test_gate_false_on_long_tensor_keeps_moments_and_moves_p():
    n = 2 * SLOTS * CHUNK + 777
    a, b = Case(n, 1), Case(5000, 2)
    run_and_check([a, b], "warm-up")
    step2 = 1e-3 * math.sqrt(1 - 0.999 ** 2) / (1 - 0.9 ** 2)
    a.step = b.step = step2
    a.set_grad(np.zeros(n))
    before = run_and_check([a, b], "zero gradient")
    assert np.array_equal(a.m.cpu().numpy().view(np.uint32), before[0][2].view(np.uint32))
    assert np.array_equal(a.v.cpu().numpy().view(np.uint32), before[0][3].view(np.uint32))
    assert not np.array_equal(a.p.cpu().numpy(), before[0][0])      # stale momentum still moves p
    assert not np.array_equal(b.m.cpu().numpy(), before[1][2])


def test_gate_opened_by_one_element_at_either_end():
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = [(SLOTS + 3) * CHUNK - 5, (SLOTS + 3) * CHUNK - 5, 2 * SLOTS * CHUNK + 1, (SLOTS + 5) * CHUNK,
             (8 * sm + SLOTS + 3) * CHUNK + 9, SLOTS * CHUNK + 3]
    where = [0, -1, -1, (SLOTS + 2) * CHUNK + 17, -1, None]          # None: the all-zero tensor
    cases = []
    for i, (n, w) in enumerate(zip(sizes, where)):
        g = np.zeros(n, F32)
        if w is not None:
            g[w] = 0.5 if i % 2 else -3.0
        cases.append(Case(n, 10 + i, grad=g, step=2e-3 * (i + 1)))
    run_and_check(cases[:5], "single element")
    run_and_check(cases[5:], "all zero")


def test_gate_with_negative_zero_weight_decay_and_grad_scale():
    n = 3 * CHUNK + 5
    cases = [Case(n, 20, grad=np.full(n, -0.0, F32)),                        # gate false
             Case(n, 21, grad=np.zeros(n, F32), wd=1e-2),                    # weight decay alone opens it
             Case(n, 22, gscale=1.0 / 3.0),
             Case(n, 23, grad=np.zeros(n, F32)),
             Case(n, 24, gscale=1.0 / 3.0, wd=5e-3)]
    before = run_and_check(cases, "gate values")
    for k in (0, 3):
        assert np.array_equal(cases[k].m.cpu().numpy().view(np.uint32), before[k][2].view(np.uint32))


def test_inf_element_opens_the_gate_and_matches_nan_positions():
    n = 2 * CHUNK + 11
    g = np.random.default_rng(30).standard_normal(n).astype(F32)
    g[5], g[CHUNK + 1] = np.inf, -np.inf
    z = np.zeros(n, F32)
    z[n - 1] = np.inf
    cases = [Case(n, 31, grad=g), Case(n, 32, grad=z)]
    run_and_check(cases, "inf")
    for c in cases:
        assert np.isnan(c.p.cpu().numpy()).sum() == np.isinf(c.g.cpu().numpy()).sum()


def test_nan_element_freezes_the_moments_of_its_tensor():
    """grad.norm() > 0 is False when any element is NaN: the reference leaves exp_avg and exp_avg_sq untouched and
    moves p with the old moments, so p stays finite."""
    n = (SLOTS + 3) * CHUNK + 5
    r = np.random.default_rng(40)
    g_mid = r.standard_normal(n).astype(F32)
    g_mid[n // 2] = np.nan
    g_last = np.zeros(n, F32)
    g_last[-1] = np.nan
    g_first = r.standard_normal(3 * SLOTS * CHUNK).astype(F32)
    g_first[0] = np.nan
    cases = [Case(n, 41, grad=g_mid), Case(n, 42, grad=g_last), Case(n, 43), Case(len(g_first), 44, grad=g_first)]
    before = run_and_check(cases, "nan")
    for k in (0, 1, 3):
        c, b = cases[k], before[k]
        assert np.array_equal(c.m.cpu().numpy().view(np.uint32), b[2].view(np.uint32)), f"tensor {k}: m moved"
        assert np.array_equal(c.v.cpu().numpy().view(np.uint32), b[3].view(np.uint32)), f"tensor {k}: v moved"
        assert np.all(np.isfinite(c.p.cpu().numpy())), f"tensor {k}: p not finite"


@pytest.mark.parametrize("offset", [0, 1], ids=["vector", "scalar"])
def test_per_point_lr_rows_straddle_float4_groups_and_blocks(offset):
    cases = []
    for i, row in enumerate((1, 3, 7, 45)):
        rows = (2 * CHUNK + 333) // row + 1 + i
        cases.append(Case(rows * row, 50 + i, row_len=row, ppl=True, offset=offset, step=3e-3 * (i + 1)))
    run_and_check(cases, f"per_point_lr offset {offset}")


@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "offset"])
def test_sizes_around_the_block(offset):
    sizes = (1, 3, 4, 2047, 2048, 2049, 4096 * 3 + 5)
    cases = [Case(n, 60 + i, offset=offset, step=1e-3 * (i + 1), gmag=10.0 ** (i - 3)) for i, n in enumerate(sizes)]
    run_and_check(cases, f"sizes offset {offset}")


def test_zero_size_tensors_first_middle_and_last():
    """Through the C ABI: PerPointAdam drops empty tensors before it launches."""
    sizes = (0, 2049, 5, 0, 4096 + 3, 1, 7 * CHUNK, 0)
    cases = [Case(n, 70 + i, step=1e-3 * (i + 1), eps=1e-8 if i % 2 else 1e-15) for i, n in enumerate(sizes)]
    cases[5].set_grad(np.zeros(1))
    run_and_check(cases, "zero-size")


def test_launch_adam_splits_more_than_eight_tensors_over_one_flags_buffer():
    sizes = (100, 2 * CHUNK + 1, 3, 5000, 64, 4 * CHUNK, 17, 2048, 999, 12345, 7)
    cases = [Case(n, 80 + i, step=1e-3 * (1 + i % 4)) for i, n in enumerate(sizes)]
    cases[9].set_grad(np.zeros(sizes[9]))                 # second launch, slot 1: slot 1 of the first was open
    before = [c.snap() for c in cases]
    flags = torch.full((8,), 12345, dtype=torch.int32, device=DEV)
    launch_adam([c.entry() for c in cases], flags)
    torch.cuda.synchronize()
    for k, (c, b) in enumerate(zip(cases, before)):
        check_step(c, b, f"launch_adam tensor {k}")
    assert np.array_equal(cases[9].m.cpu().numpy(), before[9][2])


def test_skip_word_and_device_step_sizes():
    sizes = (3 * CHUNK + 7, 5, 2 * CHUNK, 0, 100, CHUNK + 1, 4 * CHUNK, 33)
    def mk():              # distinct step sizes, tensors of several blocks, one with a per-row multiplier
        return [Case(n // 3 * 3, 90 + i, step=1e-3 * (i + 1), ppl=True, row_len=3) if i == 2
                else Case(n, 90 + i, step=1e-3 * (i + 1)) for i, n in enumerate(sizes)]
    a, b = mk(), mk()
    # a non-zero skip word: nothing moves
    before = [c.snap() for c in a]
    rc, _ = launch(a, skip=torch.ones(1, dtype=torch.int32, device=DEV))
    assert rc == 0
    for c, s in zip(a, before):
        for x, y in zip(c.snap(), s):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    # a zero skip word and host step sizes; the same launch with device step sizes gives the same bits
    rc, _ = launch(a, skip=torch.zeros(1, dtype=torch.int32, device=DEV))
    assert rc == 0
    for k, (c, s) in enumerate(zip(a, before)):
        if c.n:
            check_step(c, s, f"skip 0 tensor {k}")
    step_dev = torch.tensor([c.step for c in b], dtype=torch.float32, device=DEV)
    rc, _ = launch(b, step_dev=step_dev)
    assert rc == 0
    for ca, cb in zip(a, b):
        for x, y in zip(ca.snap(), cb.snap()):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    # more than one launch's worth of device step sizes is refused
    nine = [Case(10, 100 + i) for i in range(9)]
    with pytest.raises(GsbError):
        launch_adam([c.entry() for c in nine], torch.zeros(8, dtype=torch.int32, device=DEV),
                    step_sizes_dev=torch.ones(9, device=DEV))
    arr = (GsbAdamTensor * 9)()
    for t, c in zip(arr, nine):
        c.abi(t)
    flags = torch.zeros(16, dtype=torch.int32, device=DEV)
    assert K().gsb_adam_step_ex(9, arr, flags.data_ptr(), None, step_dev.data_ptr(), _lib.stream_ptr()) == -1
    assert K().gsb_adam_step_ex(-1, arr, flags.data_ptr(), None, None, _lib.stream_ptr()) == -1


def test_per_point_adam_50_steps_with_every_third_gradient_zero():
    torch.manual_seed(5)
    P = 1000
    xyz = torch.randn(P, 3, device=DEV, requires_grad=True)
    f_rest = torch.randn(P, 15, 3, device=DEV, requires_grad=True)
    opacity = torch.randn(P, 1, device=DEV, requires_grad=True)
    rot = torch.randn(777, 4, device=DEV, requires_grad=True)
    ppl = torch.rand(P, 1, device=DEV) * 3 + 0.25
    groups = [dict(params=[xyz], lr=1.6e-4, per_point_lr=ppl), dict(params=[f_rest], lr=2.5e-3 / 20),
              dict(params=[opacity], lr=5e-2), dict(params=[rot], lr=1e-3, weight_decay=1e-2)]
    opt = PerPointAdam(groups, lr=0.0, betas=(0.9, 0.999), eps=1e-15)
    prm = [xyz, f_rest, opacity, rot]
    lrs, wds = [1.6e-4, 2.5e-3 / 20, 5e-2, 1e-3], [0.0, 0.0, 0.0, 1e-2]
    g = torch.Generator(device=DEV).manual_seed(6)
    for t in range(1, 51):
        for x in prm:
            x.grad = torch.zeros_like(x) if t % 3 == 0 else torch.randn(x.shape, device=DEV, generator=g) * 0.1
        before = []
        for x in prm:
            st = opt.state.get(x)
            m = st["exp_avg"] if st else torch.zeros_like(x)
            v = st["exp_avg_sq"] if st else torch.zeros_like(x)
            before.append(tuple(y.detach().reshape(-1).cpu().numpy().copy() for y in (x, x.grad, m, v)))
        opt.step()
        torch.cuda.synchronize()
        for i, x in enumerate(prm):
            step = lrs[i] * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)      # old-style bias correction
            c = Case.__new__(Case)
            c.n, c.row_len, c.step = x.numel(), x.numel() // x.shape[0], step
            c.hp = dict(beta1=0.9, beta2=0.999, eps=1e-15, weight_decay=wds[i], grad_scale=1.0)
            c.c = consts(**c.hp)
            st = opt.state[x]
            c.p, c.g, c.m, c.v = (y.detach().reshape(-1) for y in (x, x.grad, st["exp_avg"], st["exp_avg_sq"]))
            c.ppl = ppl.reshape(-1) if i == 0 else None
            check_step(c, before[i], f"step {t} tensor {i}")


# ---- B. gsb_fused_rs_adam_ag with W ranks on one GPU ---------------------------------------------------------------
WIDTHS = (("xyz", 3), ("f_dc", 3), ("f_rest", 45), ("opacity", 1), ("scaling", 3), ("rotation", 4))
PPL_SEGS = ("xyz", "f_rest", "scaling")


class Ranks:
    """W replicas of a flat parameter buffer on one device, each with its own gradient buffer and shard moments;
    shard boundaries at multiples of 4 that are not multiples of 2048 and fall inside rows."""

    def __init__(self, W, P=1111, seed=0):
        self.W = W
        self.segs, self.total = flat_layout(P, WIDTHS)
        N = self.total
        gen = torch.Generator(device=DEV).manual_seed(seed)
        p0 = torch.randn(N, device=DEV, generator=gen)
        self.params = [p0.clone() for _ in range(W)]
        self.grads = [torch.empty(N, device=DEV) for _ in range(W)]
        cuts = [((N * r) // W) // 4 * 4 for r in range(W)] + [N]
        cuts = [c + 4 if 0 < c < N and c % CHUNK == 0 else c for c in cuts]
        self.bounds = list(zip(cuts[:-1], cuts[1:]))
        self.m = [torch.zeros(max(4, hi - lo), device=DEV) for lo, hi in self.bounds]
        self.v = [torch.zeros(max(4, hi - lo), device=DEV) for lo, hi in self.bounds]
        # the multipliers lie at the front of larger buffers of other values: a row index off by a segment start reads
        # wrong multipliers, not unallocated memory
        self.ppl = {s: torch.rand(N + 64, device=DEV, generator=gen) * 3 + 0.25 for s in PPL_SEGS}
        self.ref_p, self.ref_m, self.ref_v = p0.clone(), torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)
        self.names = [n for n, _ in WIDTHS]
        self.step_dev = torch.empty(8, device=DEV)
        inside = [(name, c) for c in cuts[1:-1] for name, k in WIDTHS
                  if self.segs[name][0] < c < self.segs[name][1] and (c - self.segs[name][0]) % k]
        assert inside and any(name in PPL_SEGS for name, _ in inside)

    def pieces(self, r, steps, use_dev):
        lo, hi = self.bounds[r]
        out = []
        for fi, (name, k) in enumerate(WIDTHS):
            s0, s1 = self.segs[name]
            b, e = max(lo, s0), min(hi, s1)
            if e > b:
                pc = GsbShardPiece()
                pc.begin, pc.end, pc.seg_begin = b, e, s0
                pc.per_point_lr = self.ppl[name].data_ptr() if name in PPL_SEGS else None
                pc.row_len, pc.flag_index = k, fi
                pc.step_size = 0.0 if use_dev else steps[fi]
                pc.beta1, pc.beta2, pc.eps = 0.9, 0.999, 1e-15
                out.append(pc)
        return out

    def gate(self, grads):
        arr = (GsbAdamTensor * len(WIDTHS))()
        for a, (name, k) in zip(arr, WIDTHS):
            s0, s1 = self.segs[name]
            a.param = a.exp_avg = a.exp_avg_sq = a.grad = grads[s0:s1].data_ptr()
            a.numel, a.row_len, a.grad_scale = s1 - s0, k, 1.0
        flags = torch.zeros(8, dtype=torch.int32, device=DEV)
        assert K().gsb_adam_gate(len(WIDTHS), arr, flags.data_ptr(), _lib.stream_ptr()) == 0
        return flags

    def ptrs(self, ts, extra=0):
        return (ctypes.c_void_p * self.W)(*[t.data_ptr() + (extra if i == 1 else 0) for i, t in enumerate(ts)])

    def fused(self, r, steps, use_dev, flags, skip=None, pieces=None, shard_begin=None, grads_extra=0, world=None):
        pcs = self.pieces(r, steps, use_dev) if pieces is None else pieces
        parr = (GsbShardPiece * max(1, len(pcs)))(*pcs)
        return K().gsb_fused_rs_adam_ag(self.W if world is None else world, r, self.ptrs(self.grads, grads_extra),
                                        self.ptrs(self.params), self.m[r].data_ptr(), self.v[r].data_ptr(),
                                        self.bounds[r][0] if shard_begin is None else shard_begin, len(pcs), parr,
                                        flags.data_ptr(), None if skip is None else skip.data_ptr(),
                                        1.0 / self.W, self.step_dev.data_ptr() if use_dev else None,
                                        _lib.stream_ptr())

    def step(self, steps, use_dev):
        self.step_dev[:len(WIDTHS)] = torch.tensor(steps, dtype=torch.float32)
        flags = sum(self.gate(g) for g in self.grads)                   # per-rank gates summed, as the exchange does
        for r in range(self.W):
            assert self.fused(r, steps, use_dev, flags) == 0
        gsum = self.grads[0].clone()
        for g in self.grads[1:]:
            gsum = gsum + g                                              # rank order, fp32
        arr = (GsbAdamTensor * len(WIDTHS))()
        for fi, (a, (name, k)) in enumerate(zip(arr, WIDTHS)):
            s0, s1 = self.segs[name]
            a.param, a.grad = self.ref_p[s0:s1].data_ptr(), gsum[s0:s1].data_ptr()
            a.exp_avg, a.exp_avg_sq = self.ref_m[s0:s1].data_ptr(), self.ref_v[s0:s1].data_ptr()
            a.per_point_lr = self.ppl[name].data_ptr() if name in PPL_SEGS else None
            a.numel, a.row_len, a.grad_scale = s1 - s0, k, 1.0 / self.W
            a.step_size = 0.0 if use_dev else steps[fi]
            a.beta1, a.beta2, a.eps, a.weight_decay = 0.9, 0.999, 1e-15, 0.0
        f2 = torch.zeros(8, dtype=torch.int32, device=DEV)
        assert K().gsb_adam_step_ex(len(WIDTHS), arr, f2.data_ptr(), None,
                                    self.step_dev.data_ptr() if use_dev else None, _lib.stream_ptr()) == 0
        torch.cuda.synchronize()
        return flags.cpu().numpy()

    def assert_matches_reference(self, label):
        bits = lambda t: t.view(torch.int32)
        for r in range(self.W):
            assert torch.equal(bits(self.params[r]), bits(self.ref_p)), f"{label}: replica {r} differs"
        for r, (lo, hi) in enumerate(self.bounds):
            assert torch.equal(bits(self.m[r][:hi - lo]), bits(self.ref_m[lo:hi])), f"{label}: m of rank {r}"
            assert torch.equal(bits(self.v[r][:hi - lo]), bits(self.ref_v[lo:hi])), f"{label}: v of rank {r}"

    def state(self):
        return [t.clone() for t in self.params + self.m + self.v]


@pytest.mark.parametrize("W", [2, 3, 8])
def test_fused_rs_adam_ag_equals_single_gpu_adam_on_the_summed_gradient(W):
    R = Ranks(W, seed=W)
    use_dev = W != 2
    gen = torch.Generator(device=DEV).manual_seed(100 + W)
    for t in range(1, 5):
        steps = [1e-3 * (fi + 1) * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) for fi in range(len(WIDTHS))]
        for g in R.grads:
            g.copy_(torch.randn(R.total, device=DEV, generator=gen) * 0.1)
        if t == 2:                                   # opacity: zero on every rank, its gate is shut
            s0, s1 = R.segs["opacity"]
            for g in R.grads:
                g[s0:s1] = 0
        if t == 3:                                   # rotation: a NaN on the last rank freezes its moments everywhere
            s0, s1 = R.segs["rotation"]
            R.grads[-1][s0 + 5] = float("nan")
        m_before = R.ref_m.clone()
        flags = R.step(steps, use_dev)
        R.assert_matches_reference(f"W={W} step {t}")
        if t == 2:
            assert flags[3] == 0
        if t == 3:
            s0, s1 = R.segs["rotation"]
            assert FLAG_NAN <= flags[5] and torch.equal(R.ref_m[s0:s1], m_before[s0:s1])
            assert bool(torch.isfinite(R.ref_p).all())


def test_fused_skip_word_and_refusals():
    R = Ranks(3, seed=7)
    gen = torch.Generator(device=DEV).manual_seed(8)
    for g in R.grads:
        g.copy_(torch.randn(R.total, device=DEV, generator=gen))
    steps = [1e-3] * len(WIDTHS)
    R.step_dev[:len(WIDTHS)] = 1e-3
    flags = sum(R.gate(g) for g in R.grads)
    before = R.state()
    for r in range(3):
        assert R.fused(r, steps, True, flags, skip=torch.ones(1, dtype=torch.int32, device=DEV)) == 0
    torch.cuda.synchronize()
    for a, b in zip(R.state(), before):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    good = R.pieces(1, steps, False)
    lo = R.bounds[1][0]

    def bad(**kw):
        pcs = R.pieces(1, steps, False)
        for key, val in kw.items():
            setattr(pcs[0], key, val)
        return pcs

    launches = K().gsb_launch_count()
    refused = [R.fused(1, steps, False, flags, pieces=bad(begin=good[0].begin + 1)),
               R.fused(1, steps, False, flags, pieces=bad(end=good[0].end - 2)),
               R.fused(1, steps, False, flags, pieces=bad(end=good[0].begin - 4)),
               R.fused(1, steps, False, flags, pieces=bad(begin=lo - 4)),
               R.fused(1, steps, False, flags, pieces=bad(row_len=0)),
               R.fused(1, steps, False, flags, pieces=bad(flag_index=8)),
               R.fused(1, steps, False, flags, pieces=bad(flag_index=-1)),
               R.fused(1, steps, False, flags, shard_begin=lo + 2),
               R.fused(1, steps, False, flags, grads_extra=4),
               R.fused(1, steps, False, flags, world=1),
               R.fused(1, steps, False, flags, world=9)]
    torch.cuda.synchronize()
    assert refused == [-1] * len(refused)
    assert K().gsb_launch_count() == launches
    for a, b in zip(R.state(), before):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- C. gsb_track_step_batch -----------------------------------------------------------------------------------------
B1, B2, EPS_T, WD_T = float(F32(0.9)), float(F32(0.999)), float(F32(1e-8)), float(F32(1e-4))
N_IT = 500


def track_batch(V, st, dpose, sums, step, lr_q, lr_T, loss_out=None, stride=0):
    pose, m, v, best = st
    return K().gsb_track_step_batch(V, pose.data_ptr(), dpose.data_ptr(), sums.data_ptr(), m.data_ptr(), v.data_ptr(),
                                    best.data_ptr(), None if loss_out is None else loss_out.data_ptr(), stride, step,
                                    lr_q, lr_T, 0.9, 0.999, 1e-8, 1e-4, _lib.stream_ptr())


def track_single(st, w, dpose, sums, step, lr_q, lr_T, loss_out):
    pose, m, v, best = st
    off = lambda t, k: t.data_ptr() + t.element_size() * k * w
    return K().gsb_track_step(off(pose, 7), off(dpose, 7), off(sums, 2), off(m, 7), off(v, 7), off(best, 8),
                              loss_out.data_ptr() + 4 * w, step, lr_q, lr_T, 0.9, 0.999, 1e-8, 1e-4,
                              _lib.stream_ptr())


def new_state(poses):
    V = poses.shape[0]
    best = torch.zeros(V, 8, device=DEV)
    best[:, 0] = 1e20                                   # tracking.py: the initial best loss
    best[:, 1:] = poses
    return [poses.clone(), torch.zeros(V, 7, device=DEV), torch.zeros(V, 7, device=DEV), best]


def scripted(k):
    """Losses per view at iteration k: view 0 random, view 1 has an empty mask, view 2 falls in steps of three
    equal values (a tie must not replace the candidate)."""
    r = np.random.default_rng(1000 + k)
    cnt = np.array([777.0, 0.0, 256.0])
    loss = np.array([r.uniform(0.05, 0.5), 0.0, float(max(1, 60 - k // 3))])
    return cnt, loss


def test_track_step_matches_torch_adam_over_500_steps_and_batches_equal_single_views():
    from instantsplat_b200.tracking import cosine_lr
    V = 3
    rng = np.random.default_rng(3)
    q0 = rng.standard_normal((V, 4))
    poses = torch.tensor(np.concatenate([q0 / np.linalg.norm(q0, axis=1, keepdims=True), rng.standard_normal((V, 3))],
                                        1), dtype=torch.float32, device=DEV)
    poses[0, 6] = 0.0                                   # with a zero gradient: only weight decay of a zero
    A, B, C = new_state(poses), new_state(poses), new_state(poses)
    trace = torch.full((V, N_IT), -7.0, device=DEV)
    loss_b = torch.zeros(V, device=DEV)
    mags = torch.tensor([1e-8, 1e-6, 1e-4, 1e-2, 1.0, 1e2, 0.0], dtype=torch.float64)
    qs = [torch.zeros(4, dtype=torch.float64, requires_grad=True) for _ in range(V)]
    Ts = [torch.zeros(3, dtype=torch.float64, requires_grad=True) for _ in range(V)]
    opt = torch.optim.Adam([{"params": qs, "lr": 0.001}, {"params": Ts, "lr": 0.003}], betas=(B1, B2), eps=EPS_T,
                           weight_decay=WD_T, foreach=False)
    sch = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=N_IT, eta_min=1e-4)
    best_loss = np.full(V, F32(1e20))
    best_pose = poses.cpu().numpy().copy()
    gen = torch.Generator().manual_seed(4)
    for k in range(N_IT):
        cnt, loss = scripted(k)
        sums = torch.tensor(np.stack([loss * cnt, cnt], 1), dtype=torch.float64, device=DEV)
        sign = torch.where(torch.rand(V, 7, generator=gen) < 0.5, -1.0, 1.0).double()
        raw = sign * torch.rand(V, 7, generator=gen).double().add(0.5)
        raw[0] *= mags
        raw[2] *= 1e-3
        raw = raw * torch.tensor(np.maximum(cnt, 1.0))[:, None]
        dpose = raw.float().to(DEV)
        prev = [t.cpu().numpy().copy() for t in A[:3]]
        lr_q, lr_T = cosine_lr(0.001, k, N_IT), cosine_lr(0.003, k, N_IT)
        assert track_batch(V, A, dpose, sums, k + 1, lr_q, lr_T, trace[:, k:], N_IT) == 0
        for w in range(V):
            assert track_single(B, w, dpose, sums, k + 1, lr_q, lr_T, loss_b) == 0
        assert track_batch(V, C, dpose, sums, k + 1, lr_q, lr_T) == 0
        torch.cuda.synchronize()
        for a, b, c in zip(A, B, C):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"iteration {k}: batch != single views"
            assert torch.equal(a.view(torch.int32), c.view(torch.int32)), f"iteration {k}: loss_out changes the step"
        assert torch.equal(trace[:, k], loss_b), f"iteration {k}: losses"
        assert float(trace[1, k]) == 0.0
        # torch.optim.Adam in float64 from the kernel's previous state, with CosineAnnealingLR's rates
        p_prev, m_prev, v_prev = (F64(x) for x in prev)
        for w in range(V):
            for j, (t, sl) in enumerate(((qs[w], slice(0, 4)), (Ts[w], slice(4, 7)))):
                t.data = torch.from_numpy(p_prev[w, sl].copy())
                t.grad = raw[w, sl].float().double() / cnt[w] if cnt[w] > 0 else torch.zeros(sl.stop - sl.start,
                                                                                              dtype=torch.float64)
                opt.state[t] = {"step": torch.tensor(float(k)), "exp_avg": torch.from_numpy(m_prev[w, sl].copy()),
                                "exp_avg_sq": torch.from_numpy(v_prev[w, sl].copy())}
        opt.step()
        lrs = [grp["lr"] for grp in opt.param_groups]
        sch.step()
        pose_k, m_k, v_k = (t.cpu().numpy().astype(F64) for t in A[:3])
        for w in range(V):
            for t, sl, lr in ((qs[w], slice(0, 4), lrs[0]), (Ts[w], slice(4, 7), lrs[1])):
                st = opt.state[t]
                gd = np.abs(t.grad.numpy()) + WD_T * np.abs(p_prev[w, sl])
                tm = B1 * np.abs(m_prev[w, sl]) + (1 - B1) * gd
                tv = B2 * v_prev[w, sl] + (1 - B2) * gd * gd
                bc1, bc2 = 1 - B1 ** (k + 1), math.sqrt(1 - B2 ** (k + 1))
                dmax = lr / bc1 * tm / (np.sqrt(st["exp_avg_sq"].numpy()) / bc2 + EPS_T)
                ctx = f"iteration {k} view {w}"
                assert np.all(np.abs(m_k[w, sl] - st["exp_avg"].numpy()) <= 6 * U * tm), ctx + ": exp_avg"
                assert np.all(np.abs(v_k[w, sl] - st["exp_avg_sq"].numpy()) <= 10 * U * tv), ctx + ": exp_avg_sq"
                assert np.all(np.abs(pose_k[w, sl] - t.data.numpy()) <= U * (np.abs(p_prev[w, sl]) + 24 * dmax)), \
                    ctx + ": pose"
        if k == 0:                                      # empty mask at step 1: the gradient is weight decay alone
            g1 = F32(F64(F32(WD_T)) * F64(prev[0][1]))
            assert np.array_equal(m_k[1].astype(F32), (F32(1 - B1) * g1).astype(F32))
        # the candidate: the pose after the step, keyed on the loss before it, replaced only by a strictly lower loss
        lk = trace[:, k].cpu().numpy()
        assert np.array_equal(lk, (loss * cnt / np.maximum(cnt, 1.0)).astype(F32) * (cnt > 0)), f"iteration {k}: loss"
        for w in range(V):
            if lk[w] < best_loss[w]:
                best_loss[w], best_pose[w] = lk[w], A[0][w].cpu().numpy()
        bst = A[3].cpu().numpy()
        assert np.array_equal(bst[:, 0], best_loss) and np.array_equal(bst[:, 1:], best_pose), f"iteration {k}: best"
    assert float(A[3][2, 0]) == 1.0 and float(A[3][1, 0]) == 0.0
    # the candidate of the empty-mask view is the pose after step 1; of view 2, the first pose at loss 1
    assert not torch.equal(A[3][1, 1:], A[0][1])


def test_track_step_4096_views_with_loss_stride():
    V, stride, steps = 4096, 3, 3
    rng = np.random.default_rng(9)
    poses = torch.tensor(rng.standard_normal((V, 7)), dtype=torch.float32, device=DEV)
    A, B = new_state(poses), new_state(poses)
    out = torch.full((V * stride,), -5.0, device=DEV)
    loss_b = torch.zeros(V, device=DEV)
    for k in range(steps):
        cnt = rng.integers(0, 4, V).astype(F64) * 100
        sums = torch.tensor(np.stack([rng.random(V) * cnt, cnt], 1), dtype=torch.float64, device=DEV)
        dpose = torch.tensor(rng.standard_normal((V, 7)) * 10.0 ** rng.integers(-6, 3, (V, 1)), dtype=torch.float32,
                             device=DEV)
        assert track_batch(V, A, dpose, sums, k + 1, 1e-3, 3e-3, out, stride) == 0
        for w in range(V):
            assert track_single(B, w, dpose, sums, k + 1, 1e-3, 3e-3, loss_b) == 0
        torch.cuda.synchronize()
        for a, b in zip(A, B):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        o = out.view(V, stride)
        assert torch.equal(o[:, 0], loss_b)
        assert bool((o[:, 1:] == -5.0).all())
