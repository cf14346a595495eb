"""holocron_b200.transforms.detection on the GPU. Boxes and labels from the box kernel against the reference's record
(tests/golden/det_transforms.pt) bit for bit for every chain; images against the per-image torchvision oracle
(tests/_det_transforms_oracle.py) and the fp64 resampling oracle within the bounds tests/test_gpu_transforms.py holds
the resampler to, for each dtype. Then the batching properties: launches per call, no host synchronisation for the
recipe's chains and one device-to-host copy for a RandomResizedCrop chain, any box count and batch size, strided box
and label views, nothing written past the survivors or the outputs, identical bits on a second run, and the recipe's
output through DetectionTrainer._to_cuda into a YOLO training forward."""
import warnings

import numpy as np
import pytest
import torch
from torchvision.transforms import transforms as TT

import _det_transforms_oracle as DO
import _transforms_oracle as O
from holocron_b200 import _lib
from holocron_b200.trainer import DetectionTrainer
from holocron_b200.transforms import _boxes
from holocron_b200.transforms import detection as D
from test_det_transforms_cpu import G, KEYS, _records, build, emulate, plan
from test_gpu_transforms import DEV, DTYPES, _image, check_oracle

pytestmark = pytest.mark.gpu

VOC = ["aeroplane", "bicycle", "bird", "boat", "bottle", "bus", "car", "cat", "chair", "cow", "diningtable", "dog",
       "horse", "motorbike", "person", "pottedplant", "sheep", "sofa", "train", "tvmonitor"]
NORMALIZE = TT.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])


def recipe(size=416, flip=True, jitter=True, normalize=True):
    """references/detection/train.py:116-125 (and its validation chain without flip and jitter)."""
    steps = [D.VOCTargetTransform(VOC), D.Resize((size, size))]
    steps += [D.RandomHorizontalFlip()] if flip else []
    steps += [D.convert_to_relative]
    steps += [D.ImageTransform(TT.ColorJitter(brightness=0.3, contrast=0.3, saturation=0.1, hue=0.02))] if jitter else []
    steps += [D.ImageTransform(TT.PILToTensor()), D.ImageTransform(TT.ConvertImageDtype(torch.float32))]
    return D.Compose(steps + ([D.ImageTransform(NORMALIZE)] if normalize else []))


def _cuda_target(t):
    if "boxes" not in t:
        return t
    return {"boxes": t["boxes"].to(DEV), "labels": t["labels"].to(DEV)}


@pytest.mark.parametrize("key", KEYS)
def test_boxes_match_reference(key):
    """The whole record's samples as one batch: boxes and labels bit for bit, and the generator state."""
    rec = dict(_records())[key]
    steps = [build(n, a) for n, a in rec["spec"]]
    images = [torch.zeros(3, h, w, dtype=torch.uint8, device=DEV) for (h, w), _ in rec["inputs"]]
    targets = [_cuda_target(t) for _, t in rec["inputs"]]
    torch.manual_seed(rec["seed"])
    x, out = D.Compose(steps)(images, targets)
    assert torch.equal(torch.get_rng_state(), rec["state"])
    for got, want, (size, _), img in zip(out, rec["outputs"], rec["inputs"], x):
        assert got["boxes"].is_cuda and got["boxes"].dtype == torch.float32
        assert torch.equal(got["boxes"].cpu(), want["boxes"].reshape(-1, 4)), (key, size)
        assert torch.equal(got["labels"].cpu(), want["labels"]), (key, size)
        assert tuple(img.shape[-2:]) == want["after"][-1]


def _render(inner, fold):
    """A placed, mirrored canvas of an already resized box, by indexing (0 outside)."""
    Hc, Wc = fold.canvas
    ys = torch.arange(Hc, device=inner.device)[:, None] - fold.top
    us = torch.arange(Wc, device=inner.device)
    xs = ((Wc - 1 - us) if fold.mirror else us)[None, :] - fold.left
    h, w = inner.shape[-2:]
    live = (ys >= 0) & (ys < h) & (xs >= 0) & (xs < w)
    out = inner[..., ys.clamp(0, h - 1), xs.clamp(0, w - 1)]
    return torch.where(live, out, torch.zeros_like(out))


CHAINS = [[D.RandomResizedCrop(24), D.RandomHorizontalFlip(), D.CenterCrop(20)],
          [D.Resize(30), D.CenterCrop((40, 28)), D.RandomHorizontalFlip()],
          [D.Resize((16, 24)), D.RandomHorizontalFlip()]]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("chain", range(len(CHAINS)))
def test_images_against_oracles(dtype, chain):
    """Each image within the resampler's bounds of the fp64 oracle of its fold, as torchvision's tensor chain is."""
    steps = CHAINS[chain]
    sizes = [(37, 53), (61, 20), (33, 33), (9, 13)]
    images = [_image((3, h, w), dtype, 20 * chain + k) for k, (h, w) in enumerate(sizes)]
    targets = [{"boxes": torch.tensor([[1., 2., 8., 9.]], device=DEV), "labels": torch.tensor([k], device=DEV)}
               for k in range(len(sizes))]
    for seed in range(2):
        torch.manual_seed(seed)
        x, y = D.Compose(steps)(images, targets)
        torch.manual_seed(seed)
        tv = DO.apply_batch(steps, images, targets)
        torch.manual_seed(seed)
        _, _, plans = plan(steps, sizes)
        for k, ((fold,), _) in enumerate(plans):
            src = images[k]
            if fold.box is not None:
                i, j, h, w = fold.box
                src = src[..., i:i + h, j:j + w]
            value, mag = O.resize_pad(src, fold.inner, fold.inner, "bilinear", True)
            value = _render(torch.from_numpy(value), fold).numpy()
            mag = _render(torch.from_numpy(mag), fold).numpy()
            check_oracle(x[k], value, mag, "bilinear", src)
            check_oracle(tv[k][0], value, mag, "bilinear", src)
            assert torch.equal(y[k]["boxes"], tv[k][1]["boxes"]) and torch.equal(y[k]["labels"], tv[k][1]["labels"])


def _voc_batch(n=32, seed=0):
    """n VOC-like uint8 images (sides in [300, 500]) with 1-40 objects each."""
    g = np.random.default_rng(seed)
    images, targets = [], []
    for k, (h, w) in enumerate(g.integers(300, 501, (n, 2)).tolist()):
        images.append(_image((3, h, w), torch.uint8, 1000 * seed + k))
        objs = []
        for _ in range(int(g.integers(1, 41))):
            x0, x1 = sorted(g.choice(w + 1, 2, replace=False).tolist())
            y0, y1 = sorted(g.choice(h + 1, 2, replace=False).tolist())
            objs.append({"name": VOC[int(g.integers(0, 20))], "bndbox": {"xmin": str(x0), "ymin": str(y0),
                                                                        "xmax": str(x1), "ymax": str(y1)}})
        targets.append({"annotation": {"object": objs}})
    return images, targets


def test_train_recipe_against_per_image_oracle(monkeypatch):
    """32 VOC-like images through the recipe: boxes and labels bit for bit; images before ColorJitter within a rounding
    of torchvision's; after it, bit for bit given the same jittered input."""
    images, targets = _voc_batch()
    seen = {}
    real_jitter = D.jitter

    def recording_jitter(sources, draws):
        seen["pre"] = torch.stack(list(sources)).clone()
        return real_jitter(sources, draws)
    monkeypatch.setattr(D, "jitter", recording_jitter)
    torch.manual_seed(0)
    x, y = recipe()(images, targets)
    state = torch.get_rng_state()
    assert x.shape == (32, 3, 416, 416) and x.dtype == torch.float32
    torch.manual_seed(0)
    ref = DO.apply_batch(recipe().transforms, images, targets, pre_jitter=seen["pre"])
    assert torch.equal(torch.get_rng_state(), state)
    for got, (_, want, _) in zip(y, ref):
        assert torch.equal(got["boxes"], want["boxes"]) and torch.equal(got["labels"], want["labels"])
    before = torch.stack([r[2] for r in ref])
    diff = (seen["pre"].int() - before.int()).abs()
    assert diff.max() <= 1 and (diff != 0).float().mean() < 1e-3
    assert torch.equal(x, torch.stack([r[0] for r in ref]))


def test_launches_per_call():
    images, targets = _voc_batch(8, seed=2)
    lib = _lib.lib()
    for tf, launches in ((recipe(), 4), (recipe(flip=False, jitter=False), 2),
                         (D.Compose([D.VOCTargetTransform(VOC), D.RandomResizedCrop(416), D.RandomHorizontalFlip(),
                                     D.convert_to_relative]), 2),
                         (D.Compose([D.VOCTargetTransform(VOC), D.Resize(300), D.CenterCrop(256),
                                     D.RandomHorizontalFlip(), D.CenterCrop(200), D.RandomResizedCrop(128)]), 4),
                         (D.Compose([D.VOCTargetTransform(VOC), D.convert_to_relative]), 1)):
        tf(images, targets)  # warm up
        torch.cuda.synchronize()
        lib.hb_launch_count_reset()
        tf(images, targets)
        assert lib.hb_launch_count() == launches, tf  # one per run, one for the boxes, two per jitter


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return sum("called a synchronizing CUDA operation" in str(w.message) for w in caught)


def test_host_synchronisation():
    """The recipe's chains (before torchvision's Normalize, which checks its std on the device) synchronise nothing;
    a RandomResizedCrop chain makes exactly one device-to-host copy, for the survivors' counts."""
    images, targets = _voc_batch(8, seed=4)
    train, val = D.Compose(recipe().transforms[:-1]), D.Compose(recipe(flip=False, jitter=False).transforms[:-1])
    rrc = D.Compose([D.VOCTargetTransform(VOC), D.RandomResizedCrop(416), D.RandomHorizontalFlip(),
                     D.convert_to_relative])
    for tf in (train, val, rrc):
        tf(images, targets)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        train(images, targets)
        val(images, targets)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert _syncs(lambda: rrc(images, targets)) == 1


def _random_targets(counts, seed, H=300, W=400):
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in counts:
        xy = torch.rand(n, 2, 2, generator=g) * torch.tensor([W * 1.2, H * 1.2]) - torch.tensor([W * 0.1, H * 0.1])
        boxes = torch.cat([xy.min(1).values, xy.max(1).values], 1)
        boxes[: n // 7, 2] = boxes[: n // 7, 0]  # some degenerate boxes
        out.append({"boxes": boxes.to(DEV), "labels": torch.randint(0, 20, (n,), generator=g).to(DEV)})
    return out


@pytest.mark.parametrize("counts", [[0], [1], [31], [32], [33], [5000], [0, 1, 31, 32, 33, 64, 65, 4097],
                                    [int(n) for n in np.random.default_rng(5).integers(0, 70, 256)]],
                         ids=["0", "1", "31", "32", "33", "5000", "mixed", "256-images"])
def test_box_counts_and_batch_sizes(counts):
    """Against the kernel's CPU restatement of the module's own plan, bit for bit, with order kept."""
    steps = [D.RandomResizedCrop((300, 200), scale=(0.2, 0.6)), D.RandomHorizontalFlip(), D.convert_to_relative]
    images = [torch.zeros(3, 300, 400, dtype=torch.uint8, device=DEV)] * len(counts)
    targets = _random_targets(counts, len(counts))
    torch.manual_seed(1)
    _, out = D.Compose(steps)(images, targets)
    torch.manual_seed(1)
    _, ops, plans = plan(steps, [(300, 400)] * len(counts))
    assert len(out) == len(counts)
    for got, t, (_, row) in zip(out, targets, plans):
        b, lab = emulate(t["boxes"].cpu(), t["labels"].cpu(), ops, row)
        assert torch.equal(got["boxes"].cpu(), b) and torch.equal(got["labels"].cpu(), lab)


def test_strided_views_read_in_place():
    targets = _random_targets([40, 0, 7], 11)
    strided = []
    for t in targets:
        n = t["boxes"].shape[0]
        wide = torch.full((n, 7), -1.0, device=DEV)
        wide[:, 2:6] = t["boxes"]
        lab = torch.zeros(n, 3, dtype=torch.int64, device=DEV)
        lab[:, 1] = t["labels"]
        strided.append({"boxes": wide[:, 2:6], "labels": lab[:, 1]})
    assert strided[0]["boxes"].stride() == (7, 1) and strided[0]["labels"].stride() == (3,)
    steps = [D.RandomResizedCrop(64), D.RandomHorizontalFlip(), D.convert_to_relative]
    images = [torch.zeros(3, 300, 400, dtype=torch.uint8, device=DEV)] * 3
    torch.manual_seed(2)
    _, a = D.Compose(steps)(images, strided)
    torch.manual_seed(2)
    _, b = D.Compose(steps)(images, targets)
    for u, v, t in zip(a, b, targets):
        assert torch.equal(u["boxes"], v["boxes"]) and torch.equal(u["labels"], v["labels"])
    for s, t in zip(strided, targets):  # the caller's tensors are not modified
        assert torch.equal(s["boxes"], t["boxes"])


def test_canaries():
    """Nothing is written past each image's survivors or past the outputs, and counts hold the survivors."""
    targets = _random_targets([0, 33, 5, 64], 13)
    steps = [D.RandomResizedCrop(64, scale=(0.1, 0.3)), D.RandomHorizontalFlip()]
    torch.manual_seed(4)
    segments, ops, plans = plan(steps, [(300, 400)] * 4)
    rows = np.array([row for _, row in plans], dtype=np.float32)
    total = 102
    out_b = torch.full((total + 50, 4), -7.0, device=DEV)
    out_l = torch.full((total + 50,), -7, dtype=torch.int64, device=DEV)
    boxes, labels = _boxes.transform_boxes([t["boxes"] for t in targets], [t["labels"] for t in targets], ops, rows,
                                           out_boxes=out_b, out_labels=out_l)
    start = 0
    for t, b, lab, row in zip(targets, boxes, labels, rows.tolist()):
        n = t["boxes"].shape[0]
        want_b, want_l = emulate(t["boxes"].cpu(), t["labels"].cpu(), ops, row)
        assert torch.equal(b.cpu(), want_b) and (len(b) == 0 or b.data_ptr() == out_b[start:].data_ptr())
        assert torch.equal(lab.cpu(), want_l)
        assert (out_b[start + len(b):start + n] == -7).all() and (out_l[start + len(b):start + n] == -7).all()
        start += n
    assert (out_b[total:] == -7).all() and (out_l[total:] == -7).all()


def test_second_run_same_bits():
    images, targets = _voc_batch(8, seed=3)
    runs = []
    for _ in range(2):
        torch.manual_seed(5)
        runs.append(recipe()(images, targets))
    assert torch.equal(runs[0][0], runs[1][0])
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a["boxes"], b["boxes"]) and torch.equal(a["labels"], b["labels"])


def test_recipe_output_trains_yolo():
    """The recipe's output, through DetectionTrainer._to_cuda, into a YOLOv2 training forward: finite losses."""
    from holocron_b200.models.detection import yolov2
    images, targets = _voc_batch(4, seed=6)
    torch.manual_seed(0)
    x, y = recipe()(images, targets)
    x, y = DetectionTrainer._to_cuda(list(x.unbind(0)), y)
    assert all(((t["boxes"] >= 0) & (t["boxes"] <= 1)).all() for t in y)
    model = yolov2(num_classes=len(VOC)).to(DEV).train()
    losses = model(x, y)
    assert losses and all(torch.isfinite(v).all() for v in losses.values())
    sum(losses.values()).backward()
