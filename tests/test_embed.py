"""Embedding loop (SURVEY 8 a13): wire format on CPU, device path on GPU."""
import io
import os

import numpy as np
import pytest
import torch


def test_csv_wire_format_matches_pandas():
    """compute_feats.py:80-82: DataFrame(feats).to_csv(index=False, float_format='%.4f')."""
    import pandas as pd
    from dsmil_wsi_b200.embed import format_bag_csv
    rng = np.random.default_rng(0)
    feats = (rng.standard_normal((7, 12)) * np.array([1e-5, 1, 10, 100] * 3)).astype(np.float32)
    feats[0, 0] = 0.0; feats[1, 1] = -0.00004; feats[2, 2] = 12345.678
    buf = io.StringIO()
    pd.DataFrame(list(feats)).to_csv(buf, index=False, float_format="%.4f")
    assert format_bag_csv(feats) == buf.getvalue()
    # and it parses back the way train_tcga.py:24-26 reads it
    df = pd.read_csv(io.StringIO(format_bag_csv(feats)))
    assert df.shape == (7, 12) and np.allclose(df.to_numpy(), feats, atol=5.1e-5)


def test_patch_listing_mirrors_reference_globs(tmp_path):
    from dsmil_wsi_b200.embed import list_patches
    bag = tmp_path / "cls" / "slide"
    (bag / "0_0").mkdir(parents=True)
    for n in ("1_2.jpeg", "3_4.jpg", "x.png"):
        (bag / n).write_bytes(b"")
    (bag / "0_0" / "5_6.jpeg").write_bytes(b"")
    assert sorted(os.path.basename(p) for p in list_patches(str(bag), "single")) == ["1_2.jpeg", "3_4.jpg"]
    assert [os.path.basename(p) for p in list_patches(str(bag), "high")] == ["5_6.jpeg"]
    with pytest.raises(ValueError):
        list_patches(str(bag), "tree")


@pytest.mark.gpu
def test_u8_to_float_is_to_tensor():
    import torchvision.transforms.functional as VF
    from PIL import Image
    from dsmil_wsi_b200.embed import patches_to_float
    rng = np.random.default_rng(1)
    u8 = rng.integers(0, 256, size=(5, 32, 48, 3), dtype=np.uint8)
    out = patches_to_float(torch.from_numpy(u8).cuda()).cpu()
    ref = torch.stack([VF.to_tensor(Image.fromarray(a)) for a in u8])
    assert out.shape == (5, 3, 32, 48) and torch.equal(out, ref)       # bit-identical to the reference transform


@pytest.mark.gpu
@pytest.mark.parametrize("Cc", [1, 3])
def test_u8_to_float_is_to_tensor_past_one_grid(Cc):
    """12 x 224 x 224 pixels: more than the kernel's grid covers in one sweep (kSms * 16 CTAs x 256 threads = 540 672),
    so the grid-stride loop takes a second turn."""
    import torchvision.transforms.functional as VF
    from PIL import Image
    from dsmil_wsi_b200.embed import patches_to_float
    rng = np.random.default_rng(3 + Cc)
    u8 = rng.integers(0, 256, size=(12, 224, 224, Cc), dtype=np.uint8)
    assert 12 * 224 * 224 > 132 * 16 * 256
    out = patches_to_float(torch.from_numpy(u8).cuda()).cpu()
    ref = torch.stack([VF.to_tensor(Image.fromarray(a[..., 0] if Cc == 1 else a)) for a in u8])
    assert out.shape == (12, Cc, 224, 224) and torch.equal(out, ref)


@pytest.mark.gpu
def test_embedding_loop_matches_reference_style_loop(tmp_path):
    """compute_feats(...) on synthetic JPEG patches vs the reference's loop shape (to_tensor -> .cuda() ->
    i_classifier -> .cpu()), same IClassifier (ResNet-18 + InstanceNorm as compute_feats.py:146-170)."""
    import torchvision.models as models
    import torchvision.transforms.functional as VF
    from PIL import Image
    import dsmil as mil
    from dsmil_wsi_b200.embed import compute_feats, list_patches
    rng = np.random.default_rng(2)
    bag = tmp_path / "WSI" / "ds" / "single" / "c0" / "slideA"
    bag.mkdir(parents=True)
    for i in range(37):
        Image.fromarray(rng.integers(0, 256, size=(64, 64, 3), dtype=np.uint8)).save(bag / f"{i}_{i}.jpeg", quality=70)
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = False      # compare the two loops in fp32 (TF32 conv noise is ~1e-2 here)
    resnet = models.resnet18(weights=None, norm_layer=torch.nn.InstanceNorm2d)
    resnet.fc = torch.nn.Identity()
    ic = mil.IClassifier(resnet, 512, output_class=2).cuda().eval()
    got = {}

    class A:
        batch_size, num_workers = 16, 2
    compute_feats(A(), [str(bag)], ic, save_path=str(tmp_path / "datasets" / "ds"),
                  sink=lambda d, f, c: got.update(feats=f.clone(), classes=c.clone()))
    paths = list_patches(str(bag))
    with torch.no_grad():   # the reference's loop shape: DataLoader batches of args.batch_size (compute_feats.py:69-75)
        outs = [ic(torch.stack([VF.to_tensor(Image.open(p)) for p in paths[i:i + 16]]).float().cuda())
                for i in range(0, len(paths), 16)]
        rf, rc = torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])
    assert got["feats"].shape == (37, 512) and got["classes"].shape == (37, 2)
    scale = rf.abs().max().item()
    assert (got["feats"] - rf).abs().max().item() < 1e-4 * scale        # same inputs bit for bit, same backbone
    assert (got["classes"] - rc).abs().max().item() < 1e-4 * max(rc.abs().max().item(), 1.0)
    import pandas as pd
    df = pd.read_csv(tmp_path / "datasets" / "ds" / "c0" / "slideA.csv")
    assert df.shape == (37, 512) and np.allclose(df.to_numpy(), got["feats"].cpu().numpy(), atol=6e-5)
