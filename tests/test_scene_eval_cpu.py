"""CPU: the scene-evaluation oracle against the reference's own computer_intersection / computer_symmetry
(tests/golden/scene_eval.npz), the hull principle behind the footprints, the box fallback, and the
`iou_states.txt` lines of PlausibilityAggregator."""
import os

import numpy as np
import pytest
import torch

from diffuscene_b200 import evaluate as E
from oracle import scene_eval_ref as R
from tests.cases_scene_eval import random_mesh

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scene_eval.npz")


def golden():
    g = np.load(GOLDEN)
    return {str(n): {k: g[str(n) + "/" + k] for k in ("bounds", "classes", "jids", "iou", "inter", "sym")}
            for n in g["names"]}


def same_ratio(got, want):
    return (np.isnan(got) and np.isnan(want)) or abs(float(got) - want) <= 1e-6 * abs(want)


@pytest.mark.parametrize("name", list(golden()))
def test_oracle_matches_reference(name):
    c = golden()[name]
    n, pairs, iou_sum, insec, ratio = R.intersection(c["bounds"])
    inter = c["inter"]
    assert (n, pairs) == (inter[0], inter[1])
    assert float(iou_sum) / pairs == inter[2]                 # bit-exact IoU sum (same division as the reference)
    assert float(insec) / pairs == inter[3]
    assert same_ratio(ratio, inter[4]), (ratio, inter[4])
    if n > 1:
        iou = R.iou_matrix(c["bounds"])[0]
        assert iou.dtype == np.float32 and np.array_equal(iou, c["iou"])
    assert R.symmetry(c["bounds"], c["classes"], c["jids"]) == c["sym"][0]
    assert R.symmetry(c["bounds"], c["classes"]) == c["sym"][1]


def test_goldens_cover_the_edge_cases():
    g = golden()
    assert {int(c["inter"][0]) for c in g.values()} >= {0, 1, 2, 21, 64}
    assert g["touching"]["inter"][3] == 0 and g["nested"]["inter"][3] == 1.0
    assert np.isnan(g["zero_area_pair"]["inter"][4])
    assert g["same_class_other_model"]["sym"][0] < g["same_class_other_model"]["sym"][1]


def _hull_vertices(fp):
    """The placement inputs a footprint keeps: every hull vertex at the raw y minimum and maximum."""
    half, aabb, hull = fp
    return np.concatenate([np.stack([hull[:, 0], np.full(len(hull), y), hull[:, 1]], 1) for y in (aabb[1], aabb[4])])


@pytest.mark.parametrize("seed", range(6))
def test_hull_bounds_equal_full_vertex_bounds(seed):
    rng = np.random.default_rng(seed)
    v, bbox = random_mesh(rng, 500)
    fp = E.model_footprint(v, bbox)
    assert len(fp[2]) < 60 and np.array_equal(fp[1], np.concatenate([v.min(0), v.max(0)]))
    assert np.array_equal(fp[0], R.raw_half_sizes(bbox))
    hv = _hull_vertices(fp)
    for _ in range(20):
        size = rng.uniform(0.05, 2.0, 3).astype(np.float32) * rng.choice([-1, 1], 3)
        t = rng.uniform(-3, 3, 3).astype(np.float32)
        a = np.float32(rng.uniform(-np.pi, np.pi))
        full = R.place_bounds(v, fp[0], size, t, a)
        hull = R.place_bounds(hv, fp[0], size, t, a)
        extent = np.abs(full).max()
        assert np.all(full[:3] <= full[3:])
        np.testing.assert_allclose(hull, full, rtol=0, atol=8 * np.finfo(np.float64).eps * extent)


def test_box_fallback_matches_a_mesh_that_is_its_own_box():
    rng = np.random.default_rng(7)
    for _ in range(50):
        h = rng.uniform(0.1, 2.0, 3)
        size = rng.uniform(0.05, 2.0, 3).astype(np.float32) * rng.choice([-1, 1], 3)
        t, a = rng.uniform(-3, 3, 3).astype(np.float32), np.float32(rng.uniform(-4, 4))
        mesh = R.place_bounds(R.box_vertices(h), R.raw_half_sizes(R.box_vertices(h)), size, t, a)
        box = R.place_bounds(R.box_vertices(np.abs(size)), None, size, t, a)
        np.testing.assert_allclose(mesh, box, rtol=0, atol=8 * np.finfo(np.float64).eps * np.abs(box).max())


def test_footprint_table_layout():
    rng = np.random.default_rng(1)
    fps = [E.model_footprint(*random_mesh(rng)), None, E.model_footprint(*random_mesh(rng))]
    tab = E.footprint_table(fps)
    off = tab["hull_offsets"]
    assert off.dtype == np.int32 and off[0] == 0 and off[1] == off[2] == len(fps[0][2])
    assert off[3] == len(tab["hull_xz"]) and np.array_equal(tab["hull_xz"][off[2]:], fps[2][2])
    assert np.array_equal(tab["raw_aabb"][1], np.zeros(6))


def _reference_lines(results, suffix):
    """The reference's loop (scripts/generate_diffusion.py:396-430) over computer_intersection / computer_symmetry
    results, transcribed."""
    from diffuscene_b200.stats_logger import AverageAggregator
    counter, tot_sym, tot_pairs = [], 0, 0
    NUM_OBJ, NUM_PAIRS, BOX_IOU, BOX_INSEC, OVERLAP_RATIO = [AverageAggregator() for _ in range(5)]
    lines = []
    for i, (inter, sym) in enumerate(results):
        num_objects, num_pairs, avg_iou, avg_insec, overlap_ratio = inter
        counter.append(num_objects)
        NUM_OBJ.value, NUM_PAIRS.value, BOX_IOU.value = num_objects, num_pairs, avg_iou
        BOX_INSEC.value, OVERLAP_RATIO.value = avg_insec, overlap_ratio
        tot_sym += sym
        tot_pairs += num_pairs
        lines.append("num scenes: {:d} - num objects avg: {:f} - std: {:f} - num pairs: {:f} - box iou: {:f} - box intersec: {:f} - overlap ratio: {:f} - total num symmetries: {:d} - total num pairs: {:d} "
                     .format(i + 1, NUM_OBJ.value, np.array(counter).std(), NUM_PAIRS.value, BOX_IOU.value,
                             BOX_INSEC.value, OVERLAP_RATIO.value, tot_sym, tot_pairs) + suffix)
    return lines


def test_aggregator_lines_match_reference_format():
    g = golden()
    names = [n for n in g if not np.isnan(g[n]["inter"][4])]
    stats = {k: [] for k in E.STAT_KEYS}
    for n in names:
        s = R.evaluate_scene(g[n]["bounds"], g[n]["classes"], g[n]["jids"])
        for k, v in zip(E.STAT_KEYS, s):
            stats[k].append(v)
    stats = {k: torch.tensor(np.array(v)) for k, v in stats.items()}
    # the overlap ratio may differ from the reference's in the last bits (its sum order), which can move a printed
    # digit: the lines are compared on the reference's own ratios
    stats["overlap_ratio"] = torch.tensor(np.float32([g[n]["inter"][4] for n in names]))
    want = _reference_lines([(tuple(g[n]["inter"][:2].astype(int)) + tuple(g[n]["inter"][2:]), int(g[n]["sym"][0]))
                             for n in names], "retrive only size")
    agg = E.PlausibilityAggregator(E.PlausibilityAggregator.SUFFIX_ONLYSIZE)
    half = len(names) // 2
    got = agg.update({k: v[:half] for k, v in stats.items()}) + agg.update({k: v[half:] for k, v in stats.items()})
    assert got == want
    assert got[-1].endswith("total num pairs: %d retrive only size" % agg.total_num_pairs)
    assert E.PlausibilityAggregator().update({k: v[:1] for k, v in stats.items()})[0].endswith(" retrive objfeats  ")


def test_categorical_kl_and_class_frequencies():
    cls = torch.tensor([[0, 1, 1, 3], [2, 2, 0, 1]])
    keep = torch.tensor([[True, True, False, True], [True, False, False, False]])
    f = E.class_frequencies(cls, keep, 4)
    assert f.dtype == torch.float64 and torch.equal(f, torch.tensor([0.25, 0.25, 0.25, 0.25], dtype=torch.float64))
    p, q = np.array([0.5, 0.5, 0.0]), np.array([0.25, 0.25, 0.5])
    assert E.categorical_kl(p, q) == (p * (np.log(p + 1e-6) - np.log(q + 1e-6))).sum()
    assert E.categorical_kl(f.numpy(), f.numpy()) == 0.0
