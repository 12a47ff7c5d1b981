"""Two-magnification ("tree") embedding mode (SURVEY 8f-4; compute_feats.py:84-126).

tests/golden/tree/ holds a tiny synthetic pyramid bag and what the UNMODIFIED reference loop wrote for it
(oracle/gen_tree_golden.py).  The traversal / parent gather / fusion / row order / CSV naming of
`embed.compute_tree_feats` are checked here on CPU by injecting a plain-torch `embed` callable (the product
default, `embed_bag`, needs a GPU: tests/test_zz_tree_gpu.py)."""
import argparse
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from dsmil_wsi_b200 import embed as E
from dsmil_wsi_b200 import formats as F

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tree")
BAG = os.path.join("WSI", "ds", "pyramid", "c0", "slideT")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(FIX, "expected.npz")))


class PlainEmbedder(nn.Module):
    """(feats, classes) like dsmil.IClassifier (dsmil.py:21-25), plain torch so it runs without a GPU."""

    def __init__(self, gold, prefix):
        super().__init__()
        self.feature_extractor = nn.Sequential(nn.Conv2d(3, 8, 3, stride=2), nn.InstanceNorm2d(8), nn.ReLU(),
                                               nn.AdaptiveAvgPool2d(1), nn.Flatten())
        self.fc = nn.Linear(8, 2)
        self.load_state_dict({k[len(prefix) + 1:]: torch.from_numpy(v) for k, v in gold.items()
                              if k.startswith(prefix + ".")}, strict=True)

    def forward(self, x):
        feats = self.feature_extractor(x)
        return feats.view(feats.shape[0], -1), self.fc(feats.view(feats.shape[0], -1))


def cpu_embed(paths, embedder, batch_size, num_workers):
    import torchvision.transforms.functional as VF
    from PIL import Image
    embedder.eval()
    with torch.no_grad():
        outs = [embedder(torch.stack([VF.to_tensor(Image.open(p)) for p in paths[i:i + batch_size]]))
                for i in range(0, len(paths), batch_size)]
    return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])


def expected_in_our_order(gold, key, low, high):
    """Golden rows are in the reference's listing order at generation time; listing order is a file-system
    property, so re-key by (low patch, high patch) names."""
    at = {(str(l), str(h)): i for i, (l, h) in enumerate(zip(gold["row_low"], gold["row_high"]))}
    order = [at[(os.path.basename(lp), os.path.basename(hp))] for lp, hl in zip(low, high) for hp in hl]
    assert sorted(order) == list(range(len(at)))
    return gold[key][order]


def test_traversal_finds_the_reference_pairs(gold, monkeypatch):
    monkeypatch.chdir(FIX)
    low, high = E.list_tree_patches(BAG)
    assert sorted(os.path.basename(p) for p in low) == ["0_0.jpeg", "0_1.jpeg", "1_0.jpg"]
    pairs = sorted((os.path.basename(lp), os.path.basename(hp)) for lp, hl in zip(low, high) for hp in hl)
    assert pairs == sorted((str(l), str(h)) for l, h in zip(gold["row_low"], gold["row_high"]))
    assert high[[os.path.basename(p) for p in low].index("0_1.jpeg")] == []      # a low patch with no folder
    for lp, hl in zip(low, high):                                                   # jpg listed before jpeg
        exts = [os.path.splitext(h)[1] for h in hl]
        assert exts == sorted(exts, key=lambda e: e != ".jpg")


@pytest.mark.parametrize("mode", ["fusion", "cat"])
def test_tree_loop_reproduces_reference_csv(gold, tmp_path, monkeypatch, mode):
    monkeypatch.chdir(FIX)
    low_net, high_net = PlainEmbedder(gold, "low"), PlainEmbedder(gold, "high")
    args = argparse.Namespace(batch_size=2, num_workers=0, tree_fusion=mode)
    got = {}
    E.compute_tree_feats(args, [BAG], low_net, high_net, save_path=str(tmp_path), wire="both",
                         sink=lambda d, f: got.update(bag=d, feats=f.clone()), embed=cpu_embed)
    low, high = E.list_tree_patches(BAG)
    want = expected_in_our_order(gold, f"feats_{mode}", low, high)
    assert got["bag"] == BAG and got["feats"].shape == want.shape == (5, 8 if mode == "fusion" else 16)
    # the golden CSV holds 4 decimals of the reference's fp32 result
    assert np.abs(got["feats"].numpy() - want).max() <= 5.1e-5
    csv = os.path.join(str(tmp_path), "c0", "slideT.csv")                           # compute_feats.py:123-125
    vals = F.read_bag_csv(csv)
    feats = got["feats"].numpy()
    # the CSV is exactly '%.4f' of our fp32 features ...
    assert np.array_equal(vals, np.array([[float("%.4f" % v) for v in row] for row in feats], np.float32))
    # ... and equal to the reference's 4 decimals, except where a feature lies within 2e-6 of a rounding midpoint:
    # there the fp32 results of two CPUs' convolution kernels (last bits) may round to either neighbour
    f = feats.astype(np.float64) * 1e4
    tie = np.abs(f - np.floor(f) - 0.5) < 2e-2
    w32 = want.astype(np.float32)
    assert np.all((vals == w32) | (tie & (np.abs(vals.astype(np.float64) - w32) <= 1.01e-4))), (vals, w32)
    exact, _ = F.read_bag_bin(os.path.join(str(tmp_path), "c0", "slideT.bin"))
    assert torch.equal(exact, got["feats"])
    if np.array_equal(want, gold[f"feats_{mode}"]) and np.array_equal(vals, w32):   # same listing order: same text
        assert open(csv).read() == str(gold[f"csv_{mode}"])


def test_fusion_is_the_reference_numpy_expression():
    rng = np.random.default_rng(0)
    high = rng.standard_normal((9, 6)).astype(np.float32)
    low = rng.standard_normal((4, 6)).astype(np.float32)
    parent = np.array([0, 0, 1, 3, 3, 3, 2, 0, 1])
    fus = E.fuse_tree_feats(torch.from_numpy(high), torch.from_numpy(low), torch.from_numpy(parent), "fusion")
    cat = E.fuse_tree_feats(torch.from_numpy(high), torch.from_numpy(low), torch.from_numpy(parent), "cat")
    for m in range(9):   # compute_feats.py:111-114, per row
        assert np.array_equal(fus[m].numpy(), (high[m][None] + 0.25 * low[parent[m]])[0])
        assert np.array_equal(cat[m].numpy(), np.concatenate((high[m][None], low[parent[m]][None, :]), axis=-1)[0])
    assert fus.dtype == torch.float32 and cat.shape == (9, 12)


def test_tree_mode_errors_mirror_the_reference(tmp_path, capsys):
    with pytest.raises(NotImplementedError, match="tree_fusion"):
        E.fuse_tree_feats(torch.zeros(1, 2), torch.zeros(1, 2), torch.zeros(1, dtype=torch.int64), "sum")
    with pytest.raises(NotImplementedError):
        E.compute_tree_feats(argparse.Namespace(tree_fusion="sum"), [], None, None)
    with pytest.raises(ValueError):
        E.fuse_tree_feats(torch.zeros(2, 3), torch.zeros(1, 4), torch.zeros(2, dtype=torch.int64), "cat")
    with pytest.raises(ValueError, match="wire"):
        E.compute_tree_feats(argparse.Namespace(tree_fusion="cat"), [], None, None, wire="xml")
    # a bag whose low patches have no high folders writes nothing and says so (compute_feats.py:120-121)
    from PIL import Image
    bag = tmp_path / "WSI" / "ds" / "pyramid" / "c1" / "empty"
    bag.mkdir(parents=True)
    Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(bag / "0_0.jpeg")
    called = []
    E.compute_tree_feats(argparse.Namespace(tree_fusion="cat"), [str(bag)], None, None, save_path=str(tmp_path / "o"),
                         embed=lambda *a: called.append(a))
    assert not called and "No valid patch extracted from: " + str(bag) in capsys.readouterr().out
    assert not os.path.exists(tmp_path / "o")
