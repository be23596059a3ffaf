"""CPU: the shape auto-encoder's autograd twin (networks.functional.shape_ae_forward) against the reference goldens
(tests/golden/sae_*.npz), the module's state-dict layout, the decoder grid, the fp64 kNN checker and the synthetic
shapes."""
import os

import numpy as np
import pytest
import torch

from diffuscene_b200.networks import functional as Fn
from diffuscene_b200.shape_ae import KLAutoEncoder
from diffuscene_b200.synthetic import SyntheticShapes
from tests.cases_shape_ae import SAE_CASES, ZERO_GRAD, ZERO_GRAD_BOUND, check_knn, probe, sae_points, sae_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RTOL, ATOL = 2e-4, 2e-5


@pytest.fixture(autouse=True)
def _grad_enabled():
    # other modules of the suite turn autograd off globally
    with torch.enable_grad():
        yield


def golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def model_for(name):
    case = SAE_CASES[name]
    m = KLAutoEncoder(latent_dim=case["latent_dim"], kl_weight=case["kl_weight"], num_points=case["P"])
    m.load_state_dict(sae_state_dict(m.state_dict(), case), strict=True)
    m.native_backward = False
    return m.train(case["train"])


def close(got, want, rtol=RTOL, atol=ATOL):
    np.testing.assert_allclose(np.asarray(got, np.float64), np.asarray(want, np.float64), rtol=rtol, atol=atol)


@pytest.mark.parametrize("name", list(SAE_CASES))
def test_state_dict_layout_matches_reference(name):
    g = golden(name)
    m = model_for(name)
    assert list(m.state_dict().keys()) == list(g["keys"])
    assert torch.equal(sae_points(SAE_CASES[name]), torch.from_numpy(g["points"]))


@pytest.mark.parametrize("name", list(SAE_CASES))
def test_twin_matches_golden(name):
    case, g = SAE_CASES[name], golden(name)
    m = model_for(name)
    t = m._tensors()
    pts = torch.from_numpy(g["points"])
    knn = [torch.from_numpy(k.astype(np.int64)) for k in g["knn"]]
    out = Fn.shape_ae_forward(t, pts, torch.from_numpy(g["eps"]), knn=knn, train=case["train"])
    close(out["latent"].detach(), g["latent"])
    close(out["kl"].detach(), g["kl"])
    close(out["recon"].detach(), g["recon"])
    for k, v in g.items():
        if k.startswith("rs1."):
            close(t[k[4:]].detach(), v)
    d1, d2, i1, i2 = Fn.chamfer_torch(pts, out["recon"])
    close(d1.detach(), g["dist1"])
    close(d2.detach(), g["dist2"])
    # indices: where they differ from the golden's, the chosen point is a (near-)tie at the golden's distance
    rec = out["recon"].detach()
    at = lambda src, dst, i: ((src - torch.gather(dst, 1, i.long()[..., None].expand(-1, -1, 3))) ** 2).sum(-1)
    close(at(pts, rec, i1), g["dist1"])
    close(at(rec, pts, i2), g["dist2"])
    if not case["train"]:
        return
    loss, cd, kl = Fn.shape_ae_loss(out, pts, case["kl_weight"])
    close(loss.detach(), g["loss"])
    close(cd.detach(), g["ld.loss.cd"])
    close(kl.detach(), g["ld.loss.kl"])
    loss.backward()
    for k, p in m.named_parameters():
        gr = p.grad.double()
        if k in ZERO_GRAD:
            assert gr.norm().item() < ZERO_GRAD_BOUND and float(g["gnorm." + k]) < ZERO_GRAD_BOUND, k
            continue
        pr = probe(k, gr.shape).double()
        close(gr.norm().item(), g["gnorm." + k])
        close((gr * pr).sum().item(), g["gdot." + k], atol=RTOL * float(g["gnorm." + k]) * pr.norm().item())
        if "grad." + k in g:
            close(gr, g["grad." + k], atol=ATOL * max(1.0, float(np.abs(g["grad." + k]).max())))


def test_twin_own_knn_matches_reference_knn():
    g = golden("sae_b")
    pts = torch.from_numpy(g["points"])
    assert torch.equal(Fn.knn_reference(pts.permute(0, 2, 1)), torch.from_numpy(g["knn"][0].astype(np.int64)))


def test_num_batches_tracked_counts_train_forwards():
    m = model_for("sae_a")
    pts = sae_points(SAE_CASES["sae_a"])[:2]
    m(pts)
    m.eval()
    m(pts)
    assert int(m.encoder.bn1.num_batches_tracked) == 1 and int(m.decoder.fold2.layers[4].num_batches_tracked) == 1


def test_grid_matches_numpy_meshgrid():
    xx = np.linspace(-0.3, 0.3, 45, dtype=np.float32)
    want = torch.Tensor(np.array(np.meshgrid(xx, xx))).view(2, -1)
    assert torch.equal(Fn.shape_ae_grid(), want)


def test_knn_checker():
    x = sae_points(SAE_CASES["sae_b"])[:1]
    good = Fn.knn_reference(x.permute(0, 2, 1).double())
    check_knn(x, good)
    bad = good.clone()
    bad[0, 5, 15] = int(torch.cdist(x[0, 5:6].double(), x[0].double()).argmax())      # the farthest point
    with pytest.raises(AssertionError):
        check_knn(x, bad)
    rev = good.flip(-1)
    with pytest.raises(AssertionError):
        check_knn(x, rev)
    # a tie: a duplicate of the 16th neighbour may replace it
    xt = x.clone()
    j16, j17 = int(good[0, 0, 15]), int(x.shape[1] - 1)
    xt[0, j17] = xt[0, j16]
    swapped = Fn.knn_reference(xt.permute(0, 2, 1).double())
    swapped[0, 0, 15] = j17 if int(swapped[0, 0, 15]) == j16 else j16
    check_knn(xt, swapped)


def test_synthetic_shapes_deterministic_with_duplicates():
    a, b = SyntheticShapes(8, 2048, seed=3), SyntheticShapes(8, 2048, seed=3)
    for i in range(8):
        assert torch.equal(a[i]["points"], b[i]["points"])
        p = a[i]["points"]
        assert p.shape == (2048, 3) and torch.unique(p, dim=0).shape[0] < 2048
        assert float(p.norm(dim=1).max()) <= 1.0 + 1e-6
    assert not torch.equal(a[0]["points"], SyntheticShapes(8, 2048, seed=4)[0]["points"])


def test_plain_autoencoder_is_not_ported():
    from scene_synthesis.networks.foldingnet_autoencoder import AutoEncoder
    with pytest.raises(NotImplementedError):
        AutoEncoder()
