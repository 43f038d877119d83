"""DeviceRayBatches over the video datasets' per-frame pixel subsets, with and without replacement (hr_sample_train_rows) on
the GPU: rows against the reference-order table built from generate_rays, the orders and draws against their NumPy
restatements (tests/train_order_oracle.py, tests/train_subset_oracle.py), training through it, from_config and the
refusals."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests import train_order_oracle as O
from tests import train_subset_oracle as S
from tests.cases import build_case
from tests.test_train_data_gpu import H, W, _cameras

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_subsample.npz")

N_FRAMES = 50
HW = H * W
# conf/experiment/dataset/technicolor.yaml:31-34 and neural_3d.yaml:32-35
TECHNICOLOR = dict(load_full_step=8, subsample_keyframe_step=4, subsample_keyframe_frac=0.25, subsample_frac=0.125)
NEURAL_3D = dict(load_full_step=4, subsample_keyframe_step=2, subsample_keyframe_frac=0.25, subsample_frac=0.125)


def _views(order):
    """50 frames of the three cameras of test_train_data_gpu.py (NDC and world-space, distinct cam_idx), each frame at time
    f / 49: frame-major (technicolor's training order) or video-major (neural_3d's)."""
    base = _cameras()

    def at(cam, f):
        return hb.Camera(pose=cam.pose, K=cam.K, width=W, height=H, time=f / (N_FRAMES - 1), cam_idx=cam.cam_idx,
                         use_ndc=cam.use_ndc, ndc_near=cam.ndc_near)

    if order == "technicolor":
        return [at(c, f) for f in range(N_FRAMES) for c in base]
    return [at(c, f) for c in base for f in range(N_FRAMES)]


def _images(n, seed=0):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, 256, size=(n, H, W, 3), dtype=np.uint8))


def _plan(dataset):
    frames = [f for f in range(N_FRAMES) for _ in range(3)] if dataset == "technicolor" else list(range(N_FRAMES)) * 3
    videos = None if dataset == "technicolor" else [v for v in range(3) for _ in range(N_FRAMES)]
    steps = TECHNICOLOR if dataset == "technicolor" else NEURAL_3D
    return S.plan(frames, counters=dataset, videos=videos, **steps)


def _full_rows(cams, images, c_in=8):
    coords = torch.cat([hb.generate_rays(cam, c_in=c_in) for cam in cams])
    rgb = (images.float() / 255).reshape(-1, 3).cuda()
    return coords, rgb


def _setup(dataset, image_seed=0, **kw):
    cams = _views(dataset)
    images = _images(len(cams), image_seed)
    rules = _plan(dataset)
    return cams, images, rules, hb.DeviceRayBatches(cams, images, subsample=rules, **kw)


@pytest.mark.parametrize("dataset", ["technicolor", "neural_3d"])
@pytest.mark.parametrize("c_in", [8, 6])
def test_gather_rows_is_the_reference_order_table(dataset, c_in):
    cams, images, rules, d = _setup(dataset, batch_size=4096, c_in=c_in)
    coords, rgb = _full_rows(cams, images, c_in)
    table = torch.from_numpy(S.table(rules, H, W)).cuda()  # coords[mask] of each view, views in order
    assert d.n_rows == table.numel() < coords.shape[0]
    out = d.gather_rows(torch.arange(d.n_rows), with_pixel_ids=True)
    assert torch.equal(out["pixel_ids"], table)
    assert torch.equal(out["coords"], coords[table])
    assert torch.equal(out["rgb"], rgb[table])
    assert torch.equal(out["weight"], torch.ones(d.n_rows, 1, device="cuda"))
    k = torch.from_numpy(np.random.RandomState(2).randint(0, d.n_rows, 999)).cuda()  # the reference's sampler, replayed
    out = d.gather_rows(k, with_pixel_ids=True)
    assert torch.equal(out["pixel_ids"], table[k]) and torch.equal(out["coords"], coords[table[k]])
    # the subsets differ per view kind, and NDC and world rows are both present
    assert {s for s, _ in rules} == {1, 4, 8}
    second_camera = 1 if dataset == "technicolor" else N_FRAMES
    assert not torch.equal(coords.view(-1, HW, c_in)[0, :, :6], coords.view(-1, HW, c_in)[second_camera, :, :6])


def test_a_permuted_epoch_visits_every_table_row_once_in_the_restated_order():
    cams, images, rules, d = _setup("technicolor", batch_size=5000, image_seed=1)
    coords, rgb = _full_rows(cams, images)
    table = S.table(rules, H, W)
    for seed, epoch in ((0, 0), (77, 5)):
        d.seed = seed
        d.set_epoch(epoch)
        assert len(d) == -(-d.n_rows // 5000)
        batches = [d.batch(i, with_pixel_ids=True, with_table_ids=True) for i in range(len(d))]
        assert [b["coords"].shape[0] for b in batches[:-1]] == [5000] * (len(d) - 1)
        assert batches[-1]["coords"].shape[0] == d.n_rows - 5000 * (len(d) - 1)
        k = torch.cat([b["table_ids"] for b in batches]).cpu().numpy()
        assert np.array_equal(np.sort(k), np.arange(d.n_rows))
        assert np.array_equal(k, O.order(d.n_rows, seed, epoch))
        assert np.array_equal(torch.cat([b["pixel_ids"] for b in batches]).cpu().numpy(), table[k])
    b = batches[3]
    assert torch.equal(b["coords"], coords[b["pixel_ids"]]) and torch.equal(b["rgb"], rgb[b["pixel_ids"]])


def test_replacement_batches_are_the_restated_draws():
    cams, images, rules, d = _setup("neural_3d", batch_size=4096, image_seed=2, replacement=True, num_iters=7)
    coords, rgb = _full_rows(cams, images)
    table = S.table(rules, H, W)
    assert len(d) == 7
    d.set_epoch(3)
    batches = list(d)
    assert len(batches) == 7 and all(b["coords"].shape[0] == 4096 for b in batches)
    for i in range(len(d)):
        b = d.batch(i, with_pixel_ids=True, with_table_ids=True)
        for key in batches[i]:
            assert torch.equal(b[key], batches[i][key]), key
        k = b["table_ids"].cpu().numpy()
        assert np.array_equal(k, S.draws(d.n_rows, 0, 3, np.arange(i * 4096, (i + 1) * 4096)))
        p = b["pixel_ids"].cpu().numpy()
        assert np.array_equal(p, table[k])
        v, y, x = p // HW, (p % HW) // W, p % W
        s = np.array([r[0] for r in rules])[v]
        o = np.array([r[1] for r in rules])[v]
        assert np.all((x + y + o) % s == 0)
        assert torch.equal(b["coords"], coords[b["pixel_ids"]]) and torch.equal(b["rgb"], rgb[b["pixel_ids"]])
        assert torch.equal(b["weight"], torch.ones(4096, 1, device="cuda"))
    with pytest.raises(IndexError):
        d.batch(7)


def test_an_all_whole_plan_is_bit_identical_to_the_original_batches():
    cams, images = _cameras(), _images(3)
    for seed, epoch in ((0, 0), (9, 4)):
        old = hb.DeviceRayBatches(cams, images, batch_size=1000, seed=seed)
        new = hb.DeviceRayBatches(cams, images, batch_size=1000, seed=seed, subsample=[(1, 0)] * 3)
        assert len(old) == len(new) == 9 and new.n_rows == old.n_pixels
        old.set_epoch(epoch)
        new.set_epoch(epoch)
        for i in range(len(old)):
            a, b = old.batch(i, with_pixel_ids=True), new.batch(i, with_pixel_ids=True, with_table_ids=True)
            for key in a:
                assert torch.equal(a[key], b[key]), (i, key)
            assert torch.equal(b["table_ids"], b["pixel_ids"])
        # without a plan the table is every pixel: table ids are pixel ids there too
        t = old.batch(2, with_pixel_ids=True, with_table_ids=True)
        assert torch.equal(t["table_ids"], t["pixel_ids"])
        assert torch.equal(old.gather_rows(torch.arange(50, 80))["coords"], old.gather(torch.arange(50, 80))["coords"])


def test_seeds_and_epochs_key_the_draws_and_reproduce_bit_for_bit():
    cams, images, rules, d = _setup("technicolor", batch_size=2048, image_seed=3, replacement=True, num_iters=100)
    e0 = d.batch(1, with_table_ids=True)
    d.set_epoch(1)
    e1 = d.batch(1, with_table_ids=True)
    assert not torch.equal(e0["table_ids"], e1["table_ids"])
    assert not torch.equal(e0["table_ids"], d.batch(2, with_table_ids=True)["table_ids"])
    d.set_epoch(0)
    again = d.batch(1, with_table_ids=True)
    fresh = hb.DeviceRayBatches(cams, images.cuda(), 2048, subsample=rules, replacement=True, num_iters=100)
    for other in (again, fresh.batch(1, with_table_ids=True)):
        for key in e0:
            assert torch.equal(e0[key], other[key]), key
    other_seed = hb.DeviceRayBatches(cams, images, 2048, seed=1, subsample=rules, replacement=True, num_iters=100)
    assert not torch.equal(e0["table_ids"], other_seed.batch(1, with_table_ids=True)["table_ids"])


def test_per_view_shares_follow_the_plan():
    """819,200 draws at seed 21: each view's row count against its share of the table, as a z-score.  The draws are
    deterministic (the restated draws give a largest |z| of 2.41 for this seed), so the bound is fixed."""
    cams, images, rules, d = _setup("technicolor", batch_size=4096, image_seed=4, replacement=True, num_iters=200)
    d.seed = 21
    counts = S.counts(rules, H, W)
    views = torch.cat([d.batch(i, with_pixel_ids=True)["pixel_ids"] // HW for i in range(len(d))])
    obs = torch.bincount(views, minlength=len(rules)).cpu().numpy()
    exp = counts / counts.sum() * views.numel()
    z = (obs - exp) / np.sqrt(exp)
    print(f"largest |z| over {len(rules)} views: {np.abs(z).max():.3f}")
    assert np.abs(z).max() < 3.0
    whole = np.array([s == 1 for s, _ in rules])
    assert abs(obs[whole].sum() / obs.sum() - counts[whole].sum() / counts.sum()) < 0.005


def test_training_through_replacement_batches_matches_training_on_the_host_table():
    """Five training_steps fed by replacement batches against five fed by the reference's path: a host table of the kept
    rows (built from generate_rays) indexed by the same draws.  The batches are bitwise equal, so the first loss is too; the
    later steps agree within a tolerance, because the render backward accumulates table gradients with float atomics."""
    case = build_case("technicolor_trained")
    cfg = hb.to_cfg({"model": case.model_cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000},
                     "dataset": case.dataset})
    cams, images, rules, d = _setup("technicolor", batch_size=1536, image_seed=5, replacement=True, num_iters=5)
    d.seed = 9
    coords, rgb = _full_rows(cams, images)
    table = torch.from_numpy(S.table(rules, H, W)).cuda()
    host_coords, host_rgb = coords[table].cpu(), rgb[table].cpu()  # the reference's all_inputs
    feeds = {"device": [d.batch(i) for i in range(5)], "reference": []}
    for i in range(5):
        idx = torch.from_numpy(S.draws(d.n_rows, 9, 0, np.arange(i * 1536, (i + 1) * 1536)))
        ref = {"coords": host_coords[idx].cuda(), "rgb": host_rgb[idx].cuda(), "weight": torch.ones(1536, 1, device="cuda")}
        for k in ref:
            assert torch.equal(feeds["device"][i][k], ref[k]), k
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


@pytest.mark.parametrize("dataset", ["technicolor", "neural_3d"])
def test_from_config_reads_the_shipped_keys(dataset):
    cams = _views(dataset)
    steps = TECHNICOLOR if dataset == "technicolor" else NEURAL_3D
    # conf/experiment/training/technicolor_tensorf.yaml: batch_size, sample_with_replacement, num_iters
    cfg = hb.to_cfg({"training": {"batch_size": 16384, "sample_with_replacement": True, "num_iters": 4000,
                                  "num_epochs": 40},
                     "dataset": dict(name=dataset, num_frames=N_FRAMES, **steps)})
    d = hb.DeviceRayBatches.from_config(cfg, cams, _images(len(cams)))
    rules = _plan(dataset)
    assert len(d) == 4000 and d.batch_size == 16384 and d.replacement
    assert d.subsample == [(s, o % s) for s, o in rules]
    assert d.n_rows == int(S.counts(rules, H, W).sum())
    assert d.batch(3999)["coords"].shape == (16384, 8)
    # the same plan as the reference's own table in the golden fixture (3 views or videos, 50 frames)
    g = np.load(GOLDEN)
    name = f"{dataset}_shipped_13x11"
    ids = g[f"{name}/ids"]
    assert np.array_equal(S.table(rules, 13, 11), ids)
    # without replacement: one pass over the table per epoch
    cfg["training"]["sample_with_replacement"] = False
    d = hb.DeviceRayBatches.from_config(cfg, cams, _images(len(cams)))
    assert not d.replacement and len(d) == -(-d.n_rows // 16384)


def test_malformed_plans_and_rows_give_zero_rows_and_the_c_abi_refuses():
    cams, images, rules, d = _setup("technicolor", batch_size=1000)
    lib = L.load_library()
    n = 64
    coords = torch.empty(n, 8, device="cuda")
    rgb = torch.empty(n, 3, device="cuda")
    w = torch.empty(n, 1, device="cuda")
    pids = torch.empty(n, dtype=torch.int64, device="cuda")
    tids = torch.empty(n, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    nv = len(cams)

    def call(mode=L.SAMPLE_PERMUTE, batch_index=0, batch_size=n, c_in=8, n_views=nv, height=H, n_table=None, rows=None,
             start=d._view_start, rule=d._view_rule, coords_ptr=coords.data_ptr(), start_ptr=None):
        out = C.c_int64(-1)
        rc = lib.hr_sample_train_rows(
            d.cameras.data_ptr(), n_views, d.images.data_ptr(), L.PIXEL_RGB8, height, W, c_in,
            start.data_ptr() if start_ptr is None else start_ptr, rule.data_ptr(),
            d.n_rows if n_table is None else n_table, mode, 0, 0, batch_index, batch_size,
            rows.data_ptr() if rows is not None else None, coords_ptr, rgb.data_ptr(), w.data_ptr(), pids.data_ptr(),
            tids.data_ptr(), C.byref(out), st)
        return rc, out.value, lib.hr_last_error().decode()

    n_batches = -(-d.n_rows // n)
    assert call()[:2] == (0, n)
    assert call(batch_index=n_batches - 1)[:2] == (0, d.n_rows - n * (n_batches - 1))
    assert call(mode=L.SAMPLE_REPLACE, batch_index=10 ** 9)[:2] == (0, n)
    for kw, msg in ((dict(batch_index=n_batches), "batch_index"), (dict(batch_index=-1), "batch_index"),
                    (dict(mode=L.SAMPLE_REPLACE, batch_index=-1), "batch_index"), (dict(mode=2), "mode"),
                    (dict(c_in=7), "c_in"), (dict(batch_size=0), "batch_size"), (dict(n_views=0), "image stack"),
                    (dict(height=0), "image stack"), (dict(n_table=0), "n_table"), (dict(n_table=nv * HW + 1), "n_table"),
                    (dict(coords_ptr=coords.data_ptr() + 4), "misaligned"),
                    (dict(start_ptr=d._view_start.data_ptr() + 4), "misaligned"), (dict(coords_ptr=None), "null"),
                    (dict(start_ptr=0), "null")):
        rc, got, err = call(**kw)
        assert rc != 0 and got == -1 and msg in err, (kw, err)

    def zero_rows(sel):
        assert torch.equal(w[sel], torch.zeros_like(w[sel])) and torch.equal(coords[sel], torch.zeros_like(coords[sel]))
        assert torch.equal(rgb[sel], torch.zeros_like(rgb[sel]))
        assert bool((pids[sel] == -1).all()) and bool((tids[sel] == -1).all())

    # explicit rows outside [0, n_table): zero rows of weight 0 and ids -1; the rows inside are the table's
    rows = torch.tensor([0, -1, d.n_rows - 1, d.n_rows, 2 ** 62, 5] * 10 + [1, 2, 3, 4], dtype=torch.int64, device="cuda")
    assert call(rows=rows)[:2] == (0, n)
    bad = (rows < 0) | (rows >= d.n_rows)
    zero_rows(bad)
    assert torch.equal(tids[~bad], rows[~bad]) and bool((w[~bad] == 1).all())
    # malformed plans.  A prefix that gives every view H*W rows: a rank past the view's kept pixels is a zero row, the others
    # are the view's pixel of that rank (the draws are restated, so which is which is known)
    assert call(start=torch.arange(nv + 1, dtype=torch.int64, device="cuda") * HW, mode=L.SAMPLE_REPLACE)[0] == 0
    k = S.draws(d.n_rows, 0, 0, np.arange(n))
    v, q = k // HW, k % HW
    ok = q < S.counts(rules, H, W)[v]
    assert 0 < ok.sum() < n
    ok_t = torch.from_numpy(ok).cuda()
    zero_rows(~ok_t)
    assert torch.equal(tids[ok_t].cpu(), torch.from_numpy(k[ok]))
    want = []
    for vv, qq in zip(v[ok], q[ok]):
        s, o = rules[vv]
        y, x = S.rank_to_pixel(s, o % s, H, W, np.array([qq]))
        want.append(int(vv * HW + y[0] * W + x[0]))
    assert pids[ok_t].cpu().tolist() == want and bool((w[ok_t] == 1).all())
    # strides < 1, and a prefix that does not start at 0 (rows below its first entry): every row is a zero row
    assert call(rule=torch.zeros_like(d._view_rule), mode=L.SAMPLE_REPLACE)[0] == 0
    zero_rows(torch.ones(n, dtype=torch.bool, device="cuda"))
    assert call(start=d._view_start + 100, rows=torch.arange(n, device="cuda"))[0] == 0
    zero_rows(torch.ones(n, dtype=torch.bool, device="cuda"))
    torch.cuda.synchronize()
