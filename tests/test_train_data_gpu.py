"""DeviceRayBatches / hr_sample_train_batch on the GPU: every row against generate_rays and the image, the epoch's order against
its NumPy restatement (tests/train_order_oracle.py), reproducibility, training through it, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests import train_order_oracle as O
from tests.cases import build_case
from tests.cases_rays import RAY_CASES, _pose

pytestmark = pytest.mark.gpu

W, H = 73, 41  # the size of tests/cases_rays.py's NDC camera; N = 3 * 41 * 73 = 8979 is not a power of two


def _cameras():
    """Three views of one size: the NDC and the world-space camera of tests/cases_rays.py (different pose, time, cam_idx,
    use_ndc), and a third NDC view with its own pose, time and cam_idx."""
    ndc, world = RAY_CASES["ndc_73x41"], RAY_CASES["world_50x37"]
    return [
        hb.Camera(pose=ndc["pose"], K=ndc["K"], width=W, height=H, time=ndc["time"], cam_idx=ndc["cam_idx"], use_ndc=True,
                  ndc_near=ndc["near"]),
        hb.Camera(pose=world["pose"], K=world["K"], width=W, height=H, time=world["time"], cam_idx=world["cam_idx"],
                  use_ndc=False, ndc_near=world["near"]),
        hb.Camera(pose=_pose(0.03, 0.02, [-0.1, 0.05, 0.2]), K=ndc["K"], width=W, height=H, time=30.0 / 49.0, cam_idx=1.0,
                  use_ndc=True, ndc_near=ndc["near"]),
    ]


def _images(n=3, seed=0):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, 256, size=(n, H, W, 3), dtype=np.uint8))


def _reference_rows(cams, images, c_in=8):
    """What the reference's all_inputs holds per pixel, built with the existing ray path: generate_rays of each view,
    concatenated, and T.ToTensor() of the pixels (u8 / 255 in fp32, on the host as torchvision computes it)."""
    coords = torch.cat([hb.generate_rays(cam, c_in=c_in) for cam in cams])
    rgb = (images.float() / 255).reshape(-1, 3).cuda()
    return coords, rgb


@pytest.mark.parametrize("c_in", [8, 6])
def test_rows_equal_the_existing_ray_path(c_in):
    cams, images = _cameras(), _images()
    coords, rgb = _reference_rows(cams, images, c_in)
    n = coords.shape[0]
    perm = np.random.RandomState(1).permutation(n)  # the reference's shuffle, given explicitly
    d = hb.DeviceRayBatches(cams, images, batch_size=1024, c_in=c_in)
    for ids in (torch.from_numpy(perm), torch.from_numpy(perm[:777]).cuda()):
        out = d.gather(ids, with_pixel_ids=True)
        idx = ids.cuda()
        assert torch.equal(out["coords"], coords[idx])
        assert torch.equal(out["rgb"], rgb[idx])
        assert torch.equal(out["weight"], torch.ones(idx.numel(), 1, device="cuda"))
        assert torch.equal(out["pixel_ids"], idx)
    # and through the shuffled batches: each row is its pixel's row
    for i in (0, len(d) - 1):
        out = d.batch(i, with_pixel_ids=True)
        ids = out["pixel_ids"]
        assert torch.equal(out["coords"], coords[ids]) and torch.equal(out["rgb"], rgb[ids])
    # the views really differ in what the row carries
    v = coords.view(3, H * W, c_in)
    assert not torch.equal(v[0, :, :6], v[2, :, :6]) and not torch.equal(v[0, :, :6], v[1, :, :6])
    if c_in == 8:
        assert [float(v[k, 0, 6]) for k in range(3)] == [3.0, 0.0, 1.0]
        assert len({float(v[k, 0, 7]) for k in range(3)}) == 3


def test_an_epoch_visits_every_pixel_exactly_once_in_the_restated_order():
    cams, images = _cameras(), _images()
    n = 3 * H * W
    for seed, epoch in ((0, 0), (12345, 7)):
        d = hb.DeviceRayBatches(cams, images.cuda(), batch_size=1000, seed=seed)
        d.set_epoch(epoch)
        assert len(d) == 9
        batches = [d.batch(i, with_pixel_ids=True) for i in range(len(d))]
        assert [b["coords"].shape[0] for b in batches] == [1000] * 8 + [979]  # a ragged last batch
        ids = torch.cat([b["pixel_ids"] for b in batches]).cpu().numpy()
        assert np.array_equal(np.sort(ids), np.arange(n))
        assert np.array_equal(ids, O.order(n, seed, epoch))
    it = list(d)
    assert len(it) == 9 and all(torch.equal(a["coords"], b["coords"]) for a, b in zip(it, batches))


def test_epochs_differ_and_a_seed_and_epoch_reproduce_bit_for_bit():
    cams, images = _cameras(), _images()
    d = hb.DeviceRayBatches(cams, images, batch_size=4096, seed=3)
    e0 = d.batch(1, with_pixel_ids=True)
    d.set_epoch(1)
    e1 = d.batch(1, with_pixel_ids=True)
    assert not torch.equal(e0["pixel_ids"], e1["pixel_ids"])
    d.set_epoch(0)
    again = d.batch(1, with_pixel_ids=True)
    fresh = hb.DeviceRayBatches(cams, images.cuda(), batch_size=4096, seed=3).batch(1, with_pixel_ids=True)
    for other in (again, fresh):
        for k in e0:
            assert torch.equal(e0[k], other[k]), k
    other_seed = hb.DeviceRayBatches(cams, images, batch_size=4096, seed=4).batch(1, with_pixel_ids=True)
    assert not torch.equal(e0["pixel_ids"], other_seed["pixel_ids"])


def test_training_through_device_batches_matches_training_on_the_same_rows():
    """Five training_steps fed by DeviceRayBatches against five fed by the same rows built with generate_rays and indexing.
    The batches are bitwise equal, so the first loss is too.  The steps after it are compared within a tolerance, because the
    render backward accumulates table gradients with float atomics and two runs on identical inputs differ in the last bits."""
    case = build_case("technicolor_trained")
    cfg = hb.to_cfg({"model": case.model_cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000},
                     "dataset": case.dataset})
    cams, images = _cameras(), _images(seed=5)
    coords, rgb = _reference_rows(cams, images)
    d = hb.DeviceRayBatches(cams, images, batch_size=1536, seed=9)
    feeds = {"device": [], "reference": []}
    for i in range(5):
        b = d.batch(i, with_pixel_ids=True)
        ids = b.pop("pixel_ids")
        ref = {"coords": coords[ids], "rgb": rgb[ids], "weight": torch.ones(ids.numel(), 1, device="cuda")}
        for k in ref:
            assert torch.equal(b[k], ref[k]), k
        feeds["device"].append(d.batch(i))
        feeds["reference"].append(ref)
    losses, params = {}, {}
    for name, batches in feeds.items():
        torch.manual_seed(0)  # the white-background coin flips
        system = hb.INRSystem(cfg, train_net="tc")
        system.load_state_dict(case.state_dict)
        system.cuda()
        losses[name] = [float(system.training_step(b)["train/loss"]) for b in batches]
        params[name] = {k: v.detach().clone() for k, v in system.named_parameters()}
    a, b = losses["device"], losses["reference"]
    assert a[0] == b[0], losses
    assert all(abs(x - y) <= 1e-5 * abs(y) for x, y in zip(a, b)), losses
    worst = max(float((params["device"][k] - v).abs().max()) for k, v in params["reference"].items() if v.numel() > 0)
    print(f"max |param difference| after 5 steps: {worst:.3e}")
    assert worst <= 1e-5


def test_refusals():
    cams, images = _cameras(), _images()
    d = hb.DeviceRayBatches(cams, images, batch_size=1000)
    with pytest.raises(IndexError):
        d.batch(len(d))
    with pytest.raises(ValueError, match="lie in"):
        d.gather(torch.tensor([0, 3 * H * W]))
    with pytest.raises(ValueError, match="lie in"):
        d.gather(torch.tensor([-1, 5]).cuda())
    with pytest.raises(ValueError, match="integers"):
        d.gather(torch.tensor([0.0, 1.0]))
    # the C ABI's own checks
    lib = L.load_library()
    out = torch.empty(1000, 8, device="cuda")
    rgb = torch.empty(1000, 3, device="cuda")
    w = torch.empty(1000, 1, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call(batch_index=0, c_in=8, coords=out.data_ptr(), batch_size=1000):
        n = C.c_int64(-1)
        rc = lib.hr_sample_train_batch(d.cameras.data_ptr(), 3, d.images.data_ptr(), L.PIXEL_RGB8, H, W, c_in, 0, 0,
                                       batch_index, batch_size, None, coords, rgb.data_ptr(), w.data_ptr(), None, C.byref(n), st)
        return rc, n.value, lib.hr_last_error().decode()

    assert call()[:2] == (0, 1000)
    assert call(batch_index=8)[:2] == (0, 979)
    for kw, msg in ((dict(batch_index=9), "batch_index"), (dict(batch_index=-1), "batch_index"), (dict(c_in=7), "c_in"),
                    (dict(coords=out.data_ptr() + 4), "misaligned"), (dict(batch_size=0), "batch_size"),
                    (dict(coords=None), "null")):
        rc, n, err = call(**kw)
        assert rc != 0 and n == -1 and msg in err, (kw, err)
    torch.cuda.synchronize()
