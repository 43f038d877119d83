"""The Immersive dataset's importance subsample on the device (hr_build_importance_table, hr_sample_train_mask_rows): the table
against a torch restatement built from the device's own generate_rays and against the reference's tables
(tests/golden/reference/train_importance.npz), batches with and without replacement, determinism, a full-size video, training
steps fed from from_config, and the C ABI's refusal of malformed plans."""
import ctypes as C

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests import importance_oracle as O
from tests.cases_train import build_train_case
from tests.test_fisheye_oracle import load_fisheye

pytestmark = pytest.mark.gpu

CASES = O.golden_cases()
SHIPPED = dict(load_full_step=8, subsample_keyframe_step=4, subsample_keyframe_frac=0.25, subsample_frac=0.125)


def _cameras(c):
    return [hb.Camera(pose=c["pose"][v], K=c["K"][v], width=c["W"], height=c["H"], time=c["view_times"][i],
                      cam_idx=float(c["cam_id"][v]), distortion=tuple(float(k) for k in c["distortion"][v]))
            for i, v in enumerate(c["videos"])]


def _plan(c):
    return hb.importance_subsample_plan(c["frames"], c["videos"], height=c["H"], width=c["W"], **c["steps"])


def _rows(cams, images):
    """Every pixel's row, as generate_rays and T.ToTensor() give it."""
    coords = torch.cat([hb.generate_rays(cam, c_in=8) for cam in cams])
    rgb = torch.from_numpy(images.reshape(-1, 3).astype(np.float32) / np.float32(255.0)).cuda()
    return coords, rgb


def _restated_ids(cams, images, plan, coords):
    H, W = images.shape[1:3]
    return O.table_ids(images, coords[:, 5].reshape(len(cams), H * W).cpu().numpy(), plan)


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_table_equals_the_restatement_and_the_reference(c):
    cams, plan = _cameras(c), _plan(c)
    d = hb.DeviceRayBatches(cams, c["images"], batch_size=1000, seed=1, importance=plan)
    coords, rgb = _rows(cams, c["images"])
    out = d.gather_rows(torch.arange(d.n_rows), with_pixel_ids=True)
    ids = out["pixel_ids"]
    assert torch.equal(out["coords"], coords[ids]) and torch.equal(out["rgb"], rgb[ids])
    assert bool((out["weight"] == 1).all())
    got = ids.cpu().numpy()
    assert np.array_equal(got, _restated_ids(cams, c["images"], plan, coords))
    # against the reference: only a pixel whose reference dz lies within the fisheye rays' golden tolerance of -0.05 may
    # differ; none of these cases has one
    near = np.abs(c["dz"] + np.float32(0.05)) <= 4e-6
    assert int(near.sum()) == 0
    assert np.abs(coords[:, 5].cpu().numpy() - c["dz"].reshape(-1)).max() <= 4e-6
    diff = np.setxor1d(got, c["ids"])
    assert near.reshape(-1)[diff].all()
    assert np.array_equal(got, c["ids"])
    assert np.array_equal(d.view_rows.numpy(), c["counts"])
    assert d.n_rows == int(c["counts"].sum())


def test_batches_equal_gather_of_the_same_pixels():
    c = next(c for c in CASES if c["name"] == "shipped_3v_18x24")
    cams, plan = _cameras(c), _plan(c)
    table = hb.DeviceRayBatches(cams, c["images"], batch_size=1000, importance=plan)
    all_ids = table.gather_rows(torch.arange(table.n_rows), with_pixel_ids=True)["pixel_ids"]
    for kw in ({}, {"replacement": True, "num_iters": 4}):
        d = hb.DeviceRayBatches(cams, c["images"], batch_size=700, seed=4, importance=plan, **kw)
        d.set_epoch(2)
        seen = []
        for i in range(len(d)):
            out = d.batch(i, with_pixel_ids=True, with_table_ids=True)
            t = out["table_ids"]
            assert bool((t >= 0).all()) and bool((t < d.n_rows).all())
            assert torch.equal(out["pixel_ids"], all_ids[t])
            ref = d.gather(out["pixel_ids"])
            for k in ("coords", "rgb", "weight"):
                assert torch.equal(out[k], ref[k]), k
            seen.append(t)
        if not kw:  # a permuted epoch visits every table row once
            assert torch.equal(torch.cat(seen).sort().values.cpu(), torch.arange(d.n_rows))


def test_an_all_whole_plan_equals_the_rule_plan():
    c = next(c for c in CASES if c["name"] == "other_2v_15x20")
    cams, n = _cameras(c), len(c["frames"])
    for kw in ({}, {"replacement": True, "num_iters": 3}):
        a = hb.DeviceRayBatches(cams, c["images"], batch_size=999, seed=7, importance=[None] * n, **kw)
        b = hb.DeviceRayBatches(cams, c["images"], batch_size=999, seed=7, subsample=[(1, 0)] * n, **kw)
        assert a.n_rows == b.n_rows == n * c["H"] * c["W"] and len(a) == len(b)
        assert torch.equal(a.view_rows, b.view_rows)
        for i in range(len(a)):
            x, y = a.batch(i, with_pixel_ids=True, with_table_ids=True), b.batch(i, with_pixel_ids=True, with_table_ids=True)
            for k in x:
                assert torch.equal(x[k], y[k]), k


def test_two_builds_write_the_same_bits_on_any_stream():
    c = next(c for c in CASES if c["name"] == "immersive_crop_240x320")
    cams, plan = _cameras(c), _plan(c)
    a = hb.DeviceRayBatches(cams, c["images"], batch_size=64, importance=plan)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        b = hb.DeviceRayBatches(cams, c["images"], batch_size=64, importance=plan)
    side.synchronize()
    for k in ("_view_slot", "_block_start", "_masks", "_view_rows", "_view_start"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert a.n_rows == b.n_rows == int(c["counts"].sum())


def test_a_full_size_video_equals_the_restatement():
    g = load_fisheye("immersive_1280x960")
    W, H, n_frames = int(g["W"]), int(g["H"]), 9
    cams = [hb.Camera(pose=g["pose"], K=g["K"], width=W, height=H, time=f / (n_frames - 1), cam_idx=float(g["cam_idx"]),
                      distortion=tuple(float(k) for k in g["distortion"])) for f in range(n_frames)]
    images = O.video_frames(77, n_frames, H, W)
    plan = hb.importance_subsample_plan(range(n_frames), [0] * n_frames, height=H, width=W, **SHIPPED)
    assert sum(e is not None for e in plan) == 7
    d = hb.DeviceRayBatches(cams, images, batch_size=65536, importance=plan)
    coords = torch.cat([hb.generate_rays(cam, c_in=8) for cam in cams])
    want = _restated_ids(cams, images, plan, coords)
    assert d.n_rows == want.shape[0]
    got = d.gather_rows(torch.arange(d.n_rows), with_pixel_ids=True)["pixel_ids"].cpu().numpy()
    assert np.array_equal(got, want)
    assert np.array_equal(d.view_rows.numpy(), np.bincount(want // (H * W), minlength=n_frames))


def test_training_from_config_batches_matches_training_on_gathered_rows():
    """Five training_steps of immersive_z_plane fed by from_config's replacement batches against five fed by gather_rows of
    the same table ids: the batches are bitwise equal, so the first loss is too; later steps agree within the tolerance of
    the render backward's float atomics."""
    case = build_train_case("immersive_z_plane")
    o = case.rays[0, :3].tolist()
    W, H, n_frames = 48, 36, 6
    cams = [hb.Camera(pose=[[1, 0, 0, o[0]], [0, 1, 0, o[1]], [0, 0, 1, o[2]]], K=[[30.0, 0, 23.7], [0, 30.0, 17.9], [0, 0, 1]],
                      width=W, height=H, time=f / (n_frames - 1), cam_idx=float(v), distortion=(-0.1, 0.02))
            for v in range(2) for f in range(n_frames)]
    images = np.concatenate([O.video_frames(40 + v, n_frames, H, W) for v in range(2)])
    data_cfg = hb.to_cfg({"training": {"batch_size": 1024, "sample_with_replacement": True, "num_iters": 5},
                          "dataset": dict(name="immersive", num_frames=n_frames, load_full_step=4, subsample_keyframe_step=2,
                                          subsample_keyframe_frac=0.25, subsample_frac=0.125)})
    d = hb.DeviceRayBatches.from_config(data_cfg, cams, images, seed=3)
    assert len(d) == 5 and d.importance is not None and d.importance[1] == (216, 0)
    feeds = {"device": [], "gathered": []}
    for i in range(5):
        b = d.batch(i, with_table_ids=True)
        ref = d.gather_rows(b.pop("table_ids"))
        for k in ("coords", "rgb", "weight"):
            assert torch.equal(b[k], ref[k]), k
        feeds["device"].append(b)
        feeds["gathered"].append({k: ref[k].clone() for k in ("coords", "rgb", "weight")})
    cfg = hb.to_cfg({"model": case.model_cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 5}})
    losses, params = {}, {}
    for name, batches in feeds.items():
        torch.manual_seed(0)  # the white-background coin flips
        system = hb.INRSystem(cfg, dataset=case.dataset, train_net="tc")
        system.load_state_dict(case.state_dict)
        system.cuda()
        losses[name] = [float(system.training_step(b)["train/loss"]) for b in batches]
        params[name] = {k: v.detach().clone() for k, v in system.named_parameters()}
    a, b = losses["device"], losses["gathered"]
    assert a[0] == b[0], losses
    assert all(abs(x - y) <= 1e-5 * abs(y) for x, y in zip(a, b)), losses
    # the batches are bitwise equal: what differs after five Adam steps comes from the order of the backward's float atomics
    worst = max(float((params["device"][k] - v).abs().max()) for k, v in params["gathered"].items() if v.numel() > 0)
    print(f"max |param difference| after 5 steps: {worst:.3e}")
    assert worst <= 1e-4


def test_the_c_abi_refuses_malformed_plans_and_writes_nothing():
    c = next(c for c in CASES if c["name"] == "static_1v_12x16")
    cams, plan = _cameras(c), _plan(c)
    d = hb.DeviceRayBatches(cams, c["images"], batch_size=64, importance=plan)
    lib = L.load_library()
    n, hw = len(cams), c["H"] * c["W"]
    good = np.array([(-1, -1) if e is None else e for e in plan], dtype=np.int64)
    n_slots = int((good[:, 0] >= 0).sum())
    blocks = -(-hw // 256)
    outs = {"slot": torch.full((n,), 7, dtype=torch.int32, device="cuda"),
            "block_start": torch.full((n_slots * blocks,), 7, dtype=torch.int32, device="cuda"),
            "masks": torch.full((n_slots * blocks * 8,), 7, dtype=torch.int32, device="cuda"),
            "rows": torch.full((n,), 7, dtype=torch.int64, device="cuda"),
            "start": torch.full((n + 1,), 7, dtype=torch.int64, device="cuda")}
    ws_bytes = int(lib.hr_importance_workspace_bytes(n_slots))
    ws = torch.full((ws_bytes,), 7, dtype=torch.uint8, device="cuda")

    def call(p, images=d.images.data_ptr(), start=None, ws_size=ws_bytes):
        rc = lib.hr_build_importance_table(
            d.cameras.data_ptr(), n, images, c["H"], c["W"], np.ascontiguousarray(p).ctypes.data_as(C.c_void_p),
            ws.data_ptr(), ws_size, outs["slot"].data_ptr(), outs["block_start"].data_ptr(), outs["masks"].data_ptr(),
            outs["rows"].data_ptr(), outs["start"].data_ptr() if start is None else start,
            torch.cuda.current_stream().cuda_stream)
        return rc, lib.hr_last_error().decode()

    v = int(np.flatnonzero(good[:, 0] >= 0)[0])
    cases = []
    for take, prev, msg in ((hw + 1, v - 1, "outside"), (-2, v - 1, "outside"), (1, v - 2, "previous frame"),
                            (1, v, "previous frame")):
        p = good.copy()
        p[v] = (take, prev)
        cases.append((dict(p=p), msg))
    p = good.copy()
    p[0] = (1, -1)  # the first view has no previous frame
    cases += [(dict(p=p), "previous frame"), (dict(p=good, images=None), "null"),
              (dict(p=good, start=outs["start"].data_ptr() + 4), "misaligned"), (dict(p=good, ws_size=ws_bytes - 1), "workspace")]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc != 0 and msg in err, (kw, err)
    torch.cuda.synchronize()
    for k, t in outs.items():
        assert bool((t == 7).all()), k
    assert bool((ws == 7).all())
    # the same call with the good plan builds d's table
    assert call(good)[0] == 0
    assert torch.equal(outs["start"], d._view_start) and torch.equal(outs["masks"], d._masks[:outs["masks"].numel()])
