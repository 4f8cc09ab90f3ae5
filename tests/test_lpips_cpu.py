"""LPIPS (VGG), host side (no GPU): the C ABI's new entries and scratch formula, the fp64 restatement against the
reference's own LPIPS (tests/golden/lpips.npz, made by oracle/make_golden_lpips.py), weight loading and its
refusals, and metrics.py's output layout with --lpips_weights."""
import json
import os
import re

import numpy as np
import pytest
import torch

from instantsplat_b200 import lpips as LP
from instantsplat_b200 import metrics as M
from oracle.lpips_oracle import lpips_vgg_fp64, seeded_weights, weights_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "lpips.npz")
NEW = ("gsb_lpips_scratch_bytes", "gsb_lpips_prepare", "gsb_lpips_conv3x3_relu", "gsb_lpips_maxpool2",
       "gsb_lpips_head")


@pytest.fixture(scope="module")
def seeded():
    z = np.load(GOLD)
    return seeded_weights(int(z["seed"]))


def test_entries_declared_and_exported():
    import instantsplat_b200 as I
    I._lib.build()
    header = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API\s+[\w\s\*]+?\b(gsb_\w+)\s*\(", header))
    L = I.lib()
    for name in NEW:
        assert name in declared and name in I._lib.EXPORTS and hasattr(L, name)


def test_scratch_bytes_closed_form():
    import instantsplat_b200 as I
    L = I.lib()
    for V, H, W in ((1, 16, 16), (3, 37, 53), (12, 288, 512), (4, 1080, 1920)):
        assert L.gsb_lpips_scratch_bytes(V, H, W) == 2 * (2 * V * H * W * 64 * 4) + V * 128 * 8
    assert L.gsb_lpips_scratch_bytes(0, 16, 16) == 0 and L.gsb_lpips_scratch_bytes(1, 0, 16) == 0


def test_seeded_weights_match_stored_hash(seeded):
    z = np.load(GOLD)
    assert seeded[2] == str(z["sha256"])


def test_rename_matches_reference_get_state_dict(seeded):
    z = np.load(GOLD)
    _, lin, _ = seeded
    assert list(lin) == z["lin_keys"].tolist()
    assert list(LP.rename_lin_keys(lin)) == z["lin_renamed"].tolist()


def test_oracle_matches_reference_fp64(seeded):
    z = np.load(GOLD)
    w = weights_of(seeded[0], seeded[1])
    for name in z["cases"].tolist():
        f = lambda a: torch.from_numpy(z[a]).permute(2, 0, 1)[None].float() / 255
        got, layers = lpips_vgg_fp64(f(f"x_{name}"), f(f"y_{name}"), w)
        want, want_layers = float(z[f"ref64_{name}"]), z[f"layers64_{name}"]
        assert abs(float(got[0]) - want) <= 1e-12 * abs(want), name
        assert np.allclose(layers[0].numpy(), want_layers, rtol=1e-12, atol=0), name
        if name == "same":
            assert float(got[0]) == 0.0 == want


def _write(tmp_path, vgg, lin):
    torch.save(vgg, tmp_path / LP.VGG_FILE)
    torch.save(lin, tmp_path / LP.LIN_FILE)


def test_hub_files_load(tmp_path, seeded):
    vgg, lin, _ = seeded
    full = dict(vgg)
    full["classifier.0.weight"] = torch.zeros(4, 3)          # torchvision's file also holds the classifier
    _write(tmp_path, full, lin)
    convs, lins = LP.read_weights(str(tmp_path / LP.VGG_FILE), str(tmp_path / LP.LIN_FILE))
    assert len(convs) == 13 and len(lins) == 5
    for (w, b), m in zip(convs, LP.VGG_CONV):
        assert torch.equal(w, vgg[f"features.{m}.weight"]) and torch.equal(b, vgg[f"features.{m}.bias"])
    for k, l in enumerate(lins):
        assert torch.equal(l, lin[f"lin{k}.model.1.weight"].reshape(-1))
    with pytest.raises(ValueError, match="CUDA device"):
        LP.LpipsVGG.from_dir(str(tmp_path), "cpu")


def test_weight_refusals(tmp_path, seeded):
    vgg, lin, _ = seeded
    cases = []
    for key in ("features.0.weight", "features.28.bias"):
        v = dict(vgg)
        del v[key]
        cases.append((v, lin, f"lacks {key}"))
    v = dict(vgg)
    v["features.7.weight"] = v["features.7.weight"][:, :64]
    cases.append((v, lin, r"features.7.weight has shape \(128, 64, 3, 3\), expected \(128, 128, 3, 3\)"))
    v = dict(vgg)
    v["features.2.bias"] = v["features.2.bias"].long()
    cases.append((v, lin, "features.2.bias is not a floating-point tensor"))
    l2 = dict(lin)
    del l2["lin3.model.1.weight"]
    cases.append((vgg, l2, "lacks lin3.model.1.weight"))
    l2 = dict(lin)
    l2["lin4.model.1.weight"] = l2["lin4.model.1.weight"][:, :256]
    cases.append((vgg, l2, r"4.1.weight has shape \(1, 256, 1, 1\)"))
    l2 = dict(lin)
    l2["lin5.model.1.weight"] = l2["lin4.model.1.weight"]
    cases.append((vgg, l2, "unexpected keys"))
    for i, (v, l, msg) in enumerate(cases):
        d = tmp_path / str(i)
        d.mkdir()
        _write(d, v, l)
        with pytest.raises(ValueError, match=msg):
            LP.read_weights(str(d / LP.VGG_FILE), str(d / LP.LIN_FILE))
    d = tmp_path / "one"
    d.mkdir()
    torch.save(vgg, d / LP.VGG_FILE)
    with pytest.raises(FileNotFoundError, match="vgg.pth"):
        LP.LpipsVGG.from_dir(str(d))
    with pytest.raises(FileNotFoundError, match="not found"):
        LP.LpipsVGG.from_dir(str(tmp_path / "missing"))
    (d / LP.LIN_FILE).write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="not a readable state dict"):
        LP.read_weights(str(d / LP.VGG_FILE), str(d / LP.LIN_FILE))


def test_size_refusals():
    a = torch.zeros(2, 3, 16, 16)
    assert LP.check_pair(a, a) == (2, 16, 16)
    for shape in ((1, 3, 15, 40), (1, 3, 40, 15)):
        t = torch.zeros(shape)
        with pytest.raises(ValueError, match="below 16 pixels"):
            LP.check_pair(t, t)
    with pytest.raises(ValueError, match="differ in shape"):
        LP.check_pair(a, torch.zeros(2, 3, 16, 17))
    with pytest.raises(ValueError, match=r"\[V, 3, H, W\]"):
        LP.check_pair(torch.zeros(2, 1, 16, 16), torch.zeros(2, 1, 16, 16))
    assert LP.layer_sizes(37, 53) == [(37, 53), (18, 26), (9, 13), (4, 6), (2, 3)]


def _fake_numbers(renders, gts, device="cuda"):
    return {"PSNR": torch.tensor([10.0 + float(r[0, 0, 0]) for r in renders], dtype=torch.float64),
            "SSIM": torch.tensor([float(g[0, 0, 0]) / 255 for g in gts], dtype=torch.float64)}


class _FakeNet:
    """Stands in for LpipsVGG: LPIPS = the view's render byte (0, 1, 1) / 1000."""


def _fake_lpips(renders, gts, net, device="cuda"):
    assert isinstance(net, _FakeNet)
    return torch.tensor([float(r[0, 1, 1]) / 1000 for r in renders], dtype=torch.float64)


def _tree(scene, names):
    from PIL import Image
    g = np.random.default_rng(3)
    for sub in ("renders", "gt"):
        os.makedirs(os.path.join(scene, "test", "ours_5", sub), exist_ok=True)
        for n in names:
            Image.fromarray(g.integers(0, 256, (8, 12, 3), dtype=np.uint8)).save(os.path.join(scene, "test", "ours_5", sub, n))


def test_metrics_layout_with_lpips(tmp_path, monkeypatch, capsys):
    monkeypatch.setattr(M, "image_numbers", _fake_numbers)
    monkeypatch.setattr(M, "lpips_numbers", _fake_lpips)
    built = []
    monkeypatch.setattr(LP.LpipsVGG, "from_dir", classmethod(lambda cls, p, d="cuda": built.append(p) or _FakeNet()))
    src = tmp_path / "src"
    src.mkdir()
    scene = tmp_path / "model"
    names = ["b.png", "a.png"]
    _tree(str(scene), names)
    wdir = str(tmp_path / "w")
    assert M.main(["-s", str(src), "-m", str(scene), str(scene), "--n_views", "3", "--lpips_weights", wdir]) == 0
    assert built == [wdir]                                                  # built once per run
    out = capsys.readouterr().out
    res = json.loads((scene / "results.json").read_text())["ours_5"]
    per = json.loads((scene / "per_view.json").read_text())["ours_5"]
    assert list(res) == ["SSIM", "PSNR", "LPIPS"] and list(per) == ["SSIM", "PSNR", "LPIPS"]
    from PIL import Image
    rd = lambda n: np.asarray(Image.open(scene / "test" / "ours_5" / "renders" / n))
    for n in names:
        assert per["LPIPS"][n] == float(rd(n)[0, 1, 1]) / 1000
    assert res["LPIPS"] == pytest.approx(np.mean(list(per["LPIPS"].values())), rel=1e-15)
    assert f"  LPIPS: {res['LPIPS']:>12.7f}" in out.splitlines() and "not computed" not in out
    lines = (scene / "test" / "ours_5" / "metrics.txt").read_text().splitlines()
    p, s, l = per["PSNR"]["a.png"], per["SSIM"]["a.png"], per["LPIPS"]["a.png"]
    assert lines[0] == f"image namea.png, image idx: 0, PSNR: {p:.2f}, SSIM: {s:.4f}, LPIPS: {l:.4f}"


def test_metrics_refuses_weight_dir_before_writing(tmp_path, capsys):
    scene = tmp_path / "model"
    _tree(str(scene), ["a.png"])
    with pytest.raises(SystemExit) as e:
        M.main(["-s", str(tmp_path), "-m", str(scene), "--n_views", "3", "--lpips_weights", str(tmp_path / "none")])
    assert e.value.code == 2 and "LPIPS weights" in capsys.readouterr().err
    assert not (scene / "results.json").exists() and not (scene / "test" / "ours_5" / "metrics.txt").exists()
