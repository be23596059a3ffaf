"""GPU: batched scene evaluation (ds_scene_boxes / ds_scene_stats, diffuscene_b200.evaluate) against the reference's
own computer_intersection / computer_symmetry (tests/golden/scene_eval.npz) and the fp64 full-vertex oracle."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200 import evaluate as E
from diffuscene_b200.postprocess import ObjectCatalog, post_process_batch
from oracle import retrieval_ref as RR
from oracle import scene_eval_ref as R
from tests.cases_scene_eval import random_mesh, random_scene
from tests.test_scene_eval_cpu import golden, same_ratio

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dev = torch.device("cuda")


def _stats(bounds, classes, keep=None, jids=None, pair_iou=True):
    t = lambda a, dt: None if a is None else torch.as_tensor(np.asarray(a), dtype=dt, device=dev)
    out = E.scene_stats(t(bounds, torch.float64), t(classes, torch.int64), t(keep, torch.bool), t(jids, torch.int64),
                        pair_iou=pair_iou)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _check_scene(got, b, c, with_jids=True):
    inter = c["inter"]
    n, pairs = int(got["num_objects"][b]), int(got["num_pairs"][b])
    assert (n, pairs) == (inter[0], inter[1])
    assert float(got["iou_sum"][b]) / pairs == inter[2]
    assert float(got["insec_count"][b]) / pairs == inter[3]
    assert same_ratio(got["overlap_ratio"][b], inter[4]), (got["overlap_ratio"][b], inter[4])
    assert got["num_symmetry"][b] == c["sym"][0 if with_jids else 1]


@pytest.mark.parametrize("with_jids", [True, False])
def test_stats_on_golden_bounds(with_jids):
    g = golden()
    for name, c in g.items():
        n = len(c["bounds"])
        got = _stats(c["bounds"][None], c["classes"][None], None, c["jids"][None] if with_jids else None)
        _check_scene(got, 0, c, with_jids)
        if n > 1:
            assert np.array_equal(got["pair_iou"][0], c["iou"]), name        # every pair IoU bit-equal


def test_stats_kept_objects_scattered_in_a_padded_batch():
    """All golden scenes in one [B, 64] batch, each scene's objects at random slots between dropped ones."""
    g = golden()
    rng = np.random.default_rng(5)
    B, N = len(g), 64
    bounds = rng.uniform(-5, 5, (B, N, 6))                   # dropped slots hold garbage
    classes = rng.integers(0, 4, (B, N))
    jids = rng.integers(0, 4, (B, N))
    keep = np.zeros((B, N), bool)
    slots = []
    for b, c in enumerate(g.values()):
        s = np.sort(rng.choice(N, len(c["bounds"]), replace=False))
        bounds[b, s], classes[b, s], jids[b, s], keep[b, s] = c["bounds"], c["classes"], c["jids"], True
        slots.append(s)
    got = _stats(bounds, classes, keep, jids)
    for b, c in enumerate(g.values()):
        _check_scene(got, b, c)
        s = slots[b]
        m = got["pair_iou"][b]
        if len(s) > 1:
            assert np.array_equal(m[np.ix_(s, s)], c["iou"])
        assert not m[~keep[b]].any() and not m[:, ~keep[b]].any()


def _random_batch(rng, B, N):
    bounds = np.zeros((B, N, 6))
    classes = np.zeros((B, N), np.int64)
    jids = np.zeros((B, N), np.int64)
    for b in range(B):
        bounds[b], classes[b], jids[b] = random_scene(rng, N)
    keep = rng.uniform(size=(B, N)) < 0.85
    return bounds, classes, jids, keep


@pytest.mark.parametrize("N", [12, 21])
def test_full_batch_against_oracle(N):
    rng = np.random.default_rng(N)
    B = 4096
    bounds, classes, jids, keep = _random_batch(rng, B, N)
    got = _stats(bounds, classes, keep, jids, pair_iou=False)
    bad = 0
    for b in range(B):
        k = keep[b]
        n, pairs, s, cnt, ratio, sym = R.evaluate_scene(bounds[b][k], classes[b][k], jids[b][k])
        assert (got["num_objects"][b], got["num_pairs"][b], got["insec_count"][b], got["num_symmetry"][b]) == \
            (n, pairs, cnt, sym), b
        assert got["iou_sum"][b] == s, b
        bad += not same_ratio(got["overlap_ratio"][b], ratio)
    assert bad == 0


def test_batch_independence():
    rng = np.random.default_rng(11)
    bounds, classes, jids, keep = _random_batch(rng, 4096, 21)
    full = _stats(bounds, classes, keep, jids)
    for b in (0, 1, 2047, 4095):
        one = _stats(bounds[b:b + 1], classes[b:b + 1], keep[b:b + 1], jids[b:b + 1])
        for k, v in one.items():
            assert np.array_equal(v[0], full[k][b], equal_nan=True), (b, k)


def _catalogue(rng, M=24, n_classes=5, no_footprint=(3, 7)):
    meshes = [random_mesh(rng, int(rng.integers(8, 400))) for _ in range(M)]
    fps = [None if m in no_footprint else E.model_footprint(*meshes[m]) for m in range(M)]
    labels = np.arange(M) % n_classes
    feats = rng.normal(size=(M, 32)).astype(np.float32)
    sizes = np.array([R.raw_half_sizes(bb) for _, bb in meshes], np.float32)
    ids = rng.integers(0, 6, M)
    cat = ObjectCatalog(labels, feats, sizes, n_classes=n_classes + 1, footprints=E.footprint_table(fps), model_ids=ids)
    return cat, meshes, fps, labels, feats, sizes, ids


def _oracle_bounds(meshes, fps, idx, size, t, a):
    if idx < 0 or fps[idx] is None:
        return R.place_bounds(R.box_vertices(np.abs(size)), None, size, t, a)
    v, bb = meshes[idx]
    return R.place_bounds(v, R.raw_half_sizes(bb), size, t, a)


def _assert_bounds_close(got, want):
    # R's cos / sin are float32 values: CUDA and numpy may round them differently by one float32 ulp
    scale = np.abs(want).max(-1, keepdims=True) + 1.0
    err = np.abs(got - want) / scale
    assert err.max() < 8 * 2.0 ** -24, err.max()
    assert (got[..., :3] <= got[..., 3:]).all()


def test_boxes_against_full_vertex_oracle():
    rng = np.random.default_rng(2)
    cat, meshes, fps, *_ = _catalogue(rng)
    Q = 3000
    idx = rng.integers(-1, len(meshes), Q)
    size = (rng.uniform(0.02, 2.0, (Q, 3)) * rng.choice([-1, 1], (Q, 3), p=[0.1, 0.9])).astype(np.float32)
    t = rng.uniform(-3, 3, (Q, 3)).astype(np.float32)
    a = rng.uniform(-np.pi, np.pi, (Q, 1)).astype(np.float32)
    a[:8, 0] = [0, np.pi / 2, -np.pi / 2, np.pi, -np.pi, np.pi / 4, 1e-8, 3.14159]
    T = lambda x: torch.from_numpy(x).to(dev)
    got = E.scene_boxes(T(t), T(size), T(a), T(idx), cat).cpu().numpy()
    want = np.stack([_oracle_bounds(meshes, fps, idx[q], size[q], t[q], a[q, 0]) for q in range(Q)])
    _assert_bounds_close(got, want)
    exact = np.mean(np.all(got == want, -1))
    print("bit-exact placed bounds: %.1f%%" % (100 * exact))
    boxes = E.scene_boxes(T(t), T(size), T(a)).cpu().numpy()     # no catalogue: every object is its own box
    want = np.stack([R.place_bounds(R.box_vertices(np.abs(size[q])), None, size[q], t[q], a[q, 0]) for q in range(Q)])
    _assert_bounds_close(boxes, want)


@pytest.mark.parametrize("mode", ["objfeats", "objfeats_and_size", "box", None])
def test_evaluate_samples_against_oracle_chain(tmp_path, mode):
    from scene_synthesis.networks import build_network
    from tests.test_gpu_api import _config
    from diffuscene_b200.synthetic import DEFAULT_BOUNDS
    cfg = _config(tmp_path)
    torch.manual_seed(0)
    net, _, _ = build_network(30, 23, cfg, None, device="cuda", precision="fp32")
    B = 64
    samples = net.sample(torch.zeros(B, 1, 64, 64, device=dev), 12, 62, batch_size=B, clip_denoised=True, seed=3)
    rng = np.random.default_rng(4)
    cd = net.class_dim
    cat, meshes, fps, labels, feats, sizes, ids = _catalogue(rng, M=60, n_classes=cd - 1, no_footprint=(5,))
    bounds = dict(DEFAULT_BOUNDS, objfeats=DEFAULT_BOUNDS["objfeats_32"])
    got = E.evaluate_samples(net, samples, bounds, None if mode is None else cat, mode or "box", pair_iou=True)
    got_h = {k: v.cpu().numpy() for k, v in got.items() if torch.is_tensor(v)}

    # the same chain on the CPU, one scene and one object at a time as the reference runs it
    x = samples.cpu()
    bb = net.bbox_dim
    keep = ~(x[:, :, bb + cd - 1] >= 0).numpy()
    cls = x[:, :, bb:bb + cd - 1].argmax(-1).numpy()
    # post_process_batch itself is pinned to the CPU by test_gpu_post; its device output is the oracle's input here
    world = post_process_batch({"translations": samples[:, :, :3], "sizes": samples[:, :, 3:6],
                                "angles": samples[:, :, 6:8], "objfeats": samples[:, :, bb + cd:bb + cd + 32]}, bounds)
    world = {k: v.cpu().numpy() for k, v in world.items()}
    assert np.array_equal(got_h["keep"], keep) and np.array_equal(got_h["class_index"], cls)
    for b in range(B):
        k = np.nonzero(keep[b])[0]
        if len(k) == 0:
            assert got_h["num_objects"][b] == 0 and got_h["num_pairs"][b] == 1
            continue
        if mode is None:
            idx = np.full(len(k), -1)
        else:
            m = {"objfeats_and_size": 0, "objfeats": 1, "box": 2}[mode]
            idx = RR.retrieve_batch(labels, feats, sizes, cls[b, k], world["objfeats"][b, k], world["sizes"][b, k], m)
            assert np.array_equal(got_h["model_index"][b, k], idx)
        ob = np.stack([_oracle_bounds(meshes, fps, idx[i], world["sizes"][b, o], world["translations"][b, o],
                                      world["angles"][b, o, 0]) for i, o in enumerate(k)]).reshape(-1, 6)
        _assert_bounds_close(got_h["bounds"][b, k], ob)
        jid = None if mode is None else np.where(idx >= 0, ids[idx], -1)
        n, pairs, s, cnt, ratio, sym = R.evaluate_scene(ob, cls[b, k], jid)
        assert (got_h["num_objects"][b], got_h["num_pairs"][b], got_h["insec_count"][b], got_h["num_symmetry"][b]) == \
            (n, pairs, cnt, sym), b
        # the oracle places full vertex sets: its bounds may differ in the last bits, and so may the IoU sum
        assert abs(float(got_h["iou_sum"][b]) - float(s)) <= 1e-5 * max(1.0, float(s)), b
        assert abs(float(got_h["overlap_ratio"][b]) - float(ratio)) <= 1e-5 * max(1.0, abs(float(ratio))), b
        # and on its own bounds the statistics are exact
        mine = R.evaluate_scene(got_h["bounds"][b, k], cls[b, k], jid)
        assert float(got_h["iou_sum"][b]) == float(mine[2]) and got_h["insec_count"][b] == mine[3]
    assert got_h["num_objects"].sum() == keep.sum()


def test_abi_errors():
    lib = capi.load()
    p = lambda t: C.c_void_p(t.data_ptr())
    f3 = torch.zeros(4, 3, device=dev)
    a = torch.zeros(4, device=dev)
    out = torch.empty(4, 6, dtype=torch.float64, device=dev)
    off = torch.tensor([0, 4, 4], dtype=torch.int32, device=dev)
    hull = torch.zeros(4, 2, dtype=torch.float64, device=dev)
    half = torch.ones(2, 3, dtype=torch.float64, device=dev)
    aabb = torch.zeros(2, 6, dtype=torch.float64, device=dev)
    idx = torch.tensor([0, 1, -1, 0], device=dev)

    def boxes(idx_t, off_t, **kw):
        args = dict(t=p(f3), s=p(f3), a=p(a), out=p(out))
        args.update(kw)
        return lib.ds_scene_boxes(args["t"], args["s"], args["a"], None if idx_t is None else p(idx_t), 4,
                                  None if off_t is None else p(off_t), p(hull), 4, p(half), p(aabb), 2, args["out"],
                                  None)
    assert boxes(idx, off) == 0
    torch.cuda.synchronize()
    for kw in ({"t": None}, {"s": None}, {"a": None}, {"out": None}):
        assert boxes(idx, off, **kw) == -1
    assert boxes(idx, None) == -1 and b"footprint" in lib.ds_last_error()
    assert boxes(idx, torch.tensor([0, 4, 3], dtype=torch.int32, device=dev)) == -1
    assert b"offsets" in lib.ds_last_error()
    assert boxes(idx, torch.tensor([0, 5, 5], dtype=torch.int32, device=dev)) == -1      # past the hull table
    assert boxes(torch.tensor([0, 2, -1, 0], device=dev), off) == -1
    assert b"model index" in lib.ds_last_error()
    assert boxes(torch.tensor([0, -2, -1, 0], device=dev), off) == -1
    with pytest.raises(capi.DsError):
        E.scene_boxes(f3, f3, a, torch.tensor([0, 5, 0, 0], device=dev), type("Cat", (), {"footprints": {
            "hull_offsets": off, "hull_xz": hull, "raw_half": half, "raw_aabb": aabb}})())

    bnd = torch.zeros(2, 65, 6, dtype=torch.float64, device=dev)
    cls = torch.zeros(2, 65, dtype=torch.int64, device=dev)
    o32 = torch.empty(2, dtype=torch.int32, device=dev)
    of = torch.empty(2, device=dev)

    def stats(B, N, **kw):
        ptrs = dict(bounds=p(bnd), cls=p(cls), o=p(o32), f=p(of))
        ptrs.update(kw)
        return lib.ds_scene_stats(ptrs["bounds"], None, ptrs["cls"], None, B, N, ptrs["o"], p(o32), ptrs["f"],
                                  p(o32), p(of), p(o32), None, None)
    assert stats(2, 64) == 0
    assert stats(2, 65) == -1 and b"64" in lib.ds_last_error()
    assert stats(-1, 12) == -1
    assert stats(2, 12, bounds=None) == -1 and stats(2, 12, cls=None) == -1
    assert stats(2, 12, o=None) == -1 and stats(2, 12, f=None) == -1
    with pytest.raises(capi.DsError):
        E.scene_stats(bnd, cls)
    torch.cuda.synchronize()


def test_generate_script_writes_iou_states(tmp_path):
    rng = np.random.default_rng(9)
    M = 40
    meshes = [random_mesh(rng, 200) for _ in range(M)]
    fps = E.footprint_table([E.model_footprint(*m) for m in meshes])
    np.savez(str(tmp_path / "catalogue.npz"), latents=rng.normal(size=(M, 32)).astype(np.float32),
             labels=np.arange(M) % 21, sizes=np.array([R.raw_half_sizes(bb) for _, bb in meshes], np.float32),
             model_ids=np.arange(M), **fps)
    cfg = os.path.join(ROOT, "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    out = tmp_path / "gen"
    subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "generate_diffusion.py"), cfg, str(out),
                    "--n_sequences", "6", "--batch_size", "4", "--ddim", "--ddim_steps", "5", "--compute_intersec",
                    "--catalogue", str(tmp_path / "catalogue.npz")], cwd=ROOT, env=env, check=True,
                   capture_output=True, text=True, timeout=900)
    lines = open(str(out / "iou_states.txt")).read().splitlines()
    assert len(lines) == 12                                      # objfeats and only-size lines for each scene
    for i, line in enumerate(lines):
        assert line.startswith("num scenes: %d - num objects avg: " % (i // 2 + 1))
        assert line.endswith(" retrive objfeats  " if i % 2 == 0 else " retrive only size")
        assert " - box iou: " in line and " - overlap ratio: " in line and " - total num symmetries: " in line
    assert len([f for f in os.listdir(str(out)) if f.startswith("scene_")]) == 6
