"""GPU: the shape auto-encoder (ds_shape_ae_*, ds_knn, ds_chamfer_*) against the reference goldens, fp64 brute force
and the autograd twin (networks.functional.shape_ae_forward)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200.networks import functional as Fn
from diffuscene_b200.shape_ae import KLAutoEncoder, ShapeAE, chamfer_3d, chamfer_3DDist
from tests.cases_shape_ae import SAE_CASES, ZERO_GRAD, ZERO_GRAD_BOUND, check_knn, probe, sae_points, sae_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
RTOL, ATOL = 1e-3, 1e-4
# gradients: two fp32 implementations that sum in different orders.  Measured against the goldens, the worst
# relative difference of a tensor's norm is 1.4e-4 (fold1, whose input gradient is a 512-term sum with heavy
# cancellation); small tensors whose gradient is itself a cancelling sum (mean_fc.bias) are held to an absolute floor
# of 1e-6 of the whole gradient's norm instead
GRTOL, GFLOOR = 1e-3, 1e-6
# single gradient entries: a neighbourhood or global max whose two largest inputs agree to the last bits may pick a
# different argmax in another implementation and route that entry's gradient elsewhere; measured up to 1.2e-2 of the
# tensor's largest entry against the twin at B = 16, while the norms agree within 3.2e-4
GFULL = 2e-2
dev = torch.device("cuda", 0)
ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())


@pytest.fixture(autouse=True)
def _grad_enabled_fp32():
    # other modules of the suite turn autograd off globally; the twin must run its convolutions and matmuls in fp32,
    # not TF32 (torch's default for cuDNN), to be a reference for the fp32 kernels
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    with torch.enable_grad():
        yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


def golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def close(got, want, rtol=RTOL, atol=ATOL):
    np.testing.assert_allclose(np.asarray(torch.as_tensor(got).detach().cpu().double()), np.asarray(want, np.float64),
                               rtol=rtol, atol=atol)


def model_for(name, native=True, device=dev):
    case = SAE_CASES[name]
    m = KLAutoEncoder(latent_dim=case["latent_dim"], kl_weight=case["kl_weight"], num_points=case["P"])
    m.load_state_dict(sae_state_dict(m.state_dict(), case), strict=True)
    m.native_backward = native
    return m.to(device).train(case["train"])


def grads_by_name(m, flat_grads):
    return {n: flat_grads[o:o + k] for n, o, k in m._flat_names}


def check_grads(named_grads, want_norm, want_dot, want_full, shapes):
    """named_grads: name -> flat tensor.  want_*: name -> golden / twin values."""
    floor = GFLOOR * float(np.sqrt(sum(float(want_norm[k]) ** 2 for k in shapes)))
    for k, shape in shapes.items():
        g = named_grads[k].detach().double().cpu().reshape(shape)
        if k in ZERO_GRAD:
            assert g.norm().item() < ZERO_GRAD_BOUND, k
            continue
        pr = probe(k, shape).double()
        close(g.norm().item(), want_norm[k], rtol=GRTOL, atol=floor)
        close((g * pr).sum().item(), want_dot[k], rtol=0,
              atol=GRTOL * float(want_norm[k]) * pr.norm().item() + floor * pr.norm().item())
        if k in want_full:
            w = np.asarray(want_full[k])
            close(g, w, rtol=0, atol=GFULL * max(float(np.abs(w).max()), 1e-12) + floor)


def dup_cloud(B, P, C, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(B, max(P // 2, 8), C, generator=g)
    pick = torch.randint(0, base.shape[1], (B, P), generator=g)
    return torch.gather(base, 1, pick[..., None].expand(-1, -1, C)).contiguous()


# ---- 1. Chamfer ------------------------------------------------------------------------------------------------------
def chamfer_fp64(a, b, i1, i2):
    """dist1, dist2 in fp64 at the given indices, differentiable w.r.t. a and b."""
    pb = torch.gather(b, 1, i1.long()[..., None].expand(-1, -1, 3))
    pa = torch.gather(a, 1, i2.long()[..., None].expand(-1, -1, 3))
    return ((a - pb) ** 2).sum(-1), ((b - pa) ** 2).sum(-1)


@pytest.mark.parametrize("n,m", [(2048, 2025), (1000, 37), (16, 2048)])
def test_chamfer_against_fp64(n, m):
    a = dup_cloud(3, n, 3, n).to(dev)
    b = dup_cloud(3, m, 3, m + 1).to(dev)
    d1, d2, i1, i2 = chamfer_3d(a, b)
    full = ((a.double()[:, :, None] - b.double()[:, None]) ** 2).sum(-1)
    m1, m2 = full.min(dim=2).values, full.min(dim=1).values
    close(d1, m1.cpu(), rtol=1e-5, atol=1e-7)
    close(d2, m2.cpu(), rtol=1e-5, atol=1e-7)
    at1 = torch.gather(full, 2, i1.long()[..., None])[..., 0]
    at2 = torch.gather(full, 1, i2.long()[:, None, :])[:, 0]
    assert bool((at1 <= m1 * (1 + 1e-5) + 1e-9).all()) and bool((at2 <= m2 * (1 + 1e-5) + 1e-9).all())
    # backward against autograd of the fp64 restatement at the same indices, and bit-identical across runs
    g1, g2 = torch.rand(3, n, device=dev), torch.rand(3, m, device=dev)
    a64, b64 = a.double().requires_grad_(), b.double().requires_grad_()
    e1, e2 = chamfer_fp64(a64, b64, i1, i2)
    ((e1 * g1.double()).sum() + (e2 * g2.double()).sum()).backward()
    runs = []
    for _ in range(2):
        aa, bb = a.clone().requires_grad_(), b.clone().requires_grad_()
        o1, o2, _, _ = chamfer_3DDist()(aa, bb)
        ((o1 * g1).sum() + (o2 * g2).sum()).backward()
        runs.append((aa.grad.clone(), bb.grad.clone()))
    for got, want in ((runs[0][0], a64.grad), (runs[0][1], b64.grad)):
        close(got, want.cpu(), rtol=0, atol=1e-5 * float(want.abs().max()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_chamfer_against_golden():
    g = golden("sae_a")
    a, b = torch.from_numpy(g["points"]).to(dev), torch.from_numpy(g["recon"]).to(dev)
    d1, d2, i1, i2 = chamfer_3d(a, b)
    close(d1, g["dist1"], rtol=1e-5, atol=1e-7)
    close(d2, g["dist2"], rtol=1e-5, atol=1e-7)
    # where an index differs from the golden's, the point it names is a tie at the golden's distance
    e1, e2 = chamfer_fp64(a.double(), b.double(), i1, i2)
    close(e1, g["dist1"], rtol=1e-5, atol=1e-7)
    close(e2, g["dist2"], rtol=1e-5, atol=1e-7)


# ---- 2. kNN ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C_", [3, 64, 128])
@pytest.mark.parametrize("P", [2048, 1000, 16])
def test_knn_fp64_checker(C_, P):
    x = dup_cloud(2, P, C_, 7 * P + C_).to(dev)
    idx = torch.empty(2, P, 16, dtype=torch.int32, device=dev)
    lib = capi.load()
    capi.check(lib.ds_knn(ptr(x), 2, P, C_, ptr(idx), None))
    torch.cuda.synchronize()
    # fp32 accumulation over C channels: rounding up to ~C * 2^-24 relative
    check_knn(x.cpu(), idx.cpu(), rtol=1e-6 if C_ == 3 else 1e-5)


# ---- 3. parity with the goldens, kNN and eps injected ----------------------------------------------------------------
def test_parity_train_case_a():
    case, g = SAE_CASES["sae_a"], golden("sae_a")
    m = model_for("sae_a")
    ae = m._ensure_flat()
    ae.set_knn(torch.from_numpy(g["knn"].astype(np.int32)))
    pts, eps = torch.from_numpy(g["points"]).to(dev), torch.from_numpy(g["eps"]).to(dev)
    flat0 = m._flat.clone()
    kl, lat, rec = ae.forward(m._flat, pts, eps, train=True)
    close(lat, g["latent"]), close(kl, g["kl"]), close(rec, g["recon"])
    named = dict(zip([n for n, _, _ in m._flat_names], [m._flat[o:o + k] for _, o, k in m._flat_names]))
    for k, v in g.items():
        if k.startswith("rs1."):
            close(named[k[4:]], v.reshape(-1))
    d1, d2, _, _ = chamfer_3d(pts, rec)
    close(d1, g["dist1"]), close(d2, g["dist2"])
    m._flat.copy_(flat0)
    losses = ae.train_step(m._flat, m._flat_grads, pts, eps, case["kl_weight"]).cpu()
    close(losses[0], g["loss"]), close(losses[1], g["ld.loss.cd"]), close(losses[2], g["ld.loss.kl"])
    shapes = {k: p.shape for k, p in m.named_parameters()}
    full = {k[5:]: v for k, v in g.items() if k.startswith("grad.")}
    check_grads(grads_by_name(m, m._flat_grads), {k: g["gnorm." + k] for k in shapes},
                {k: g["gdot." + k] for k in shapes}, full, shapes)
    # the running statistics get no gradient
    for n, o, k in m._flat_names:
        if "running" in n:
            assert not bool(m._flat_grads[o:o + k].any())
    ae.set_knn(None)


def test_parity_eval_case_b():
    g = golden("sae_b")
    m = model_for("sae_b")
    ae = m._ensure_flat()
    ae.set_knn(torch.from_numpy(g["knn"].astype(np.int32)))
    flat0 = m._flat.clone()
    kl, lat, rec = ae.forward(m._flat, torch.from_numpy(g["points"]), torch.from_numpy(g["eps"]), train=False)
    close(lat, g["latent"]), close(kl, g["kl"]), close(rec, g["recon"])
    assert torch.equal(m._flat, flat0)      # eval mode leaves the running statistics alone
    ae.set_knn(None)


# ---- 4. native kNN inside the network --------------------------------------------------------------------------------
def test_native_knn_in_network_and_twin_replay():
    B = 16
    case = dict(SAE_CASES["sae_a"], B=B)
    m = model_for("sae_a")
    ae = m._ensure_flat()
    pts = sae_points(dict(case, seed=21)).to(dev)
    eps = torch.randn(B, case["latent_dim"], generator=torch.Generator().manual_seed(5)).to(dev)
    t_twin = {k: v.detach().clone() for k, v in m._tensors().items()}
    losses = ae.train_step(m._flat, m._flat_grads, pts, eps, case["kl_weight"]).cpu()
    knn = ae.get_knn(B).long()
    params = {k: (v.requires_grad_() if "running" not in k else v) for k, v in t_twin.items()}
    out = Fn.shape_ae_forward(params, pts, eps, knn=list(knn), train=True)
    check_knn(pts.cpu(), knn[0].cpu())
    for s in (1, 2):
        check_knn(out["knn_inputs"][s].cpu(), knn[s].cpu(), rtol=1e-4)
    loss, cd, kl = Fn.shape_ae_loss(out, pts, case["kl_weight"])
    close(losses[0], loss.item()), close(losses[1], cd.item()), close(losses[2], kl.item())
    loss.backward()
    shapes = {k: p.shape for k, p in m.named_parameters()}
    tw = {k: params[k].grad.double().cpu() for k in shapes}
    check_grads(grads_by_name(m, m._flat_grads), {k: tw[k].norm().item() for k in shapes},
                {k: (tw[k] * probe(k, shapes[k]).double()).sum().item() for k in shapes}, tw, shapes)
    named = {n: m._flat[o:o + k] for n, o, k in m._flat_names}
    for k, v in params.items():
        if "running" in k:
            close(named[k], v.reshape(-1).cpu())


# ---- 5. eval-mode batch independence ---------------------------------------------------------------------------------
def test_eval_batch_independence():
    m = model_for("sae_a").eval()
    ae = m._ensure_flat()
    pts = sae_points(dict(SAE_CASES["sae_a"], B=64, seed=33)).to(dev)
    eps = torch.randn(64, 32, generator=torch.Generator().manual_seed(6)).to(dev)
    kl, lat, rec = ae.forward(m._flat, pts, eps, train=False)
    kl1, lat1, rec1 = ae.forward(m._flat, pts[37:38], eps[37:38], train=False)
    assert torch.equal(kl[37:38], kl1) and torch.equal(lat[37:38], lat1) and torch.equal(rec[37:38], rec1)


# ---- 6. train_on_batch with NativeAdam against the twin and torch.optim.Adam -----------------------------------------
def test_train_on_batch_native_adam_against_twin():
    from diffuscene_b200.optim import NativeAdam
    from scene_synthesis.networks.foldingnet_autoencoder import train_on_batch
    from scene_synthesis.stats_logger import StatsLogger
    lr, B = 1e-4, 16
    config = {"training": {"max_grad_norm": 10.0}}
    m = model_for("sae_a")
    t = {k: v.detach().clone() for k, v in m._tensors().items()}
    ptw = [t[k].requires_grad_() for k, _ in m.named_parameters()]
    opt = NativeAdam(m.parameters(), lr=lr)
    topt = torch.optim.Adam(ptw, lr=lr)
    for step in range(3):
        pts = sae_points(dict(SAE_CASES["sae_a"], B=B, seed=40 + step)).to(dev)
        torch.manual_seed(100 + step)
        StatsLogger.instance().clear()      # the logger averages every value set since the last clear()
        train_on_batch(m, opt, {"points": pts}, config)
        log = {k: StatsLogger.instance()[k].value for k in ("loss.cd", "loss.kl", "gradnorm", "lr")}
        knn = m._ae.get_knn(B).long()
        torch.manual_seed(100 + step)
        eps = torch.randn((B, 32)).to(dev)
        topt.zero_grad()
        out = Fn.shape_ae_forward(t, pts, eps, knn=list(knn), train=True)
        loss, cd, kl = Fn.shape_ae_loss(out, pts, m.kl_weight)
        loss.backward()
        gn = torch.nn.utils.clip_grad_norm_(ptw, 10.0)
        topt.step()
        close(log["loss.cd"], cd.item()), close(log["loss.kl"], kl.item())
        close(log["gradnorm"], gn.item(), rtol=1e-3, atol=0)
        assert log["lr"] == lr
    # Adam moves an entry by about lr whatever its gradient's size, so entries whose gradient is rounding noise (the
    # biases in ZERO_GRAD, and single entries of others) may move apart by up to 2 lr per step
    for k, p in m.named_parameters():
        close(p, t[k].detach().cpu(), rtol=0, atol=6 * lr)
    assert int(m.encoder.bn1.num_batches_tracked) == 3


# ---- 7. state-dict round trip ----------------------------------------------------------------------------------------
def test_state_dict_round_trip(tmp_path):
    src = model_for("sae_b", native=False, device="cpu")
    path = str(tmp_path / "model_00000")
    torch.save(src.state_dict(), path)
    m = KLAutoEncoder(latent_dim=64, num_points=1000)
    m.load_state_dict(torch.load(path), strict=True)
    m.to(dev).train()
    for k, v in src.state_dict().items():
        assert torch.equal(m.state_dict()[k].cpu(), v), k
    pts = sae_points(SAE_CASES["sae_b"]).to(dev)
    m(pts)
    m.get_loss({"points": pts})[0].backward()
    assert int(m.decoder.fold1.layers[1].num_batches_tracked) == 2
    sd = m.state_dict()
    assert list(sd.keys()) == list(src.state_dict().keys())
    KLAutoEncoder(latent_dim=64, num_points=1000).load_state_dict({k: v.cpu() for k, v in sd.items()}, strict=True)


# ---- 8. ABI errors ---------------------------------------------------------------------------------------------------
def test_abi_errors():
    lib = capi.load()
    h = C.c_void_p()
    for F_, P in ((0, 2048), (513, 2048), (32, 15)):
        cfg = capi.DsShapeAeConfig()
        cfg.latent_dim, cfg.num_points, cfg.device = F_, P, 0
        assert lib.ds_shape_ae_create(C.byref(cfg), C.byref(h)) == -1 and not h.value
    x = torch.zeros(1, 32, 5, device=dev)
    idx = torch.zeros(1, 32, 16, dtype=torch.int32, device=dev)
    assert lib.ds_knn(ptr(x), 1, 32, 5, ptr(idx), None) == -1
    assert lib.ds_knn(ptr(x), 1, 15, 3, ptr(idx), None) == -1
    assert lib.ds_knn(None, 1, 32, 3, ptr(idx), None) == -1
    assert lib.ds_chamfer_forward(None, 4, ptr(x), 4, 1, ptr(x), ptr(x), ptr(idx), ptr(idx), None) == -1
    ae = ShapeAE(32, 64)
    with pytest.raises(capi.DsError):
        ae.get_knn(1)                                  # no kept pass yet
    flat = torch.zeros(sum(n for _, n in ae.expected_weights()), device=dev)
    pts, eps = torch.zeros(1, 64, 3, device=dev), torch.zeros(1, 32, device=dev)
    assert lib.ds_shape_ae_train_step(ae.h, ptr(flat), ptr(pts), 1, ptr(eps), 0.001, None, ptr(eps), None) == -1
    assert lib.ds_shape_ae_forward(ae.h, ptr(flat), ptr(pts), 1, None, 0, 0, None, None, None, None) == -1
    ae.forward(flat, pts, eps, train=False, keep=False)
    with pytest.raises(capi.DsError):
        ae.get_knn(1)                                  # the last pass was not kept
    ae.close()


# ---- 9. the scripts --------------------------------------------------------------------------------------------------
def test_scripts_synthetic(tmp_path):
    from diffuscene_b200.postprocess import ObjectCatalog
    cfg = os.path.join(ROOT, "config", "obj_autoencoder", "bedrooms_lat32.yaml")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    run = lambda args: subprocess.run([sys.executable] + args, cwd=ROOT, env=env, check=True, capture_output=True,
                                      text=True, timeout=900)
    run([os.path.join(ROOT, "scripts", "train_objautoencoder.py"), cfg, str(tmp_path), "--experiment_tag", "t",
         "--synthetic_objects", "32", "--num_points", "256", "--max_epochs", "1"])
    ckpt = os.path.join(str(tmp_path), "t", "model_00000")
    assert os.path.exists(ckpt)
    out = run([os.path.join(ROOT, "scripts", "generate_objautoencoder.py"), cfg, str(tmp_path / "gen"), "--weight_file",
               ckpt, "--synthetic_objects", "24", "--num_points", "256"])
    assert "scale factor:" in out.stdout
    cat = np.load(str(tmp_path / "gen" / "catalogue.npz"))
    assert cat["latents"].shape == (24, 32) and cat["labels"].shape == (24,) and cat["sizes"].shape == (24, 3)
    assert np.load(str(tmp_path / "gen" / "objfeats" / "00000.npz"))["latent"].shape == (32,)
    c = ObjectCatalog(torch.from_numpy(cat["labels"]), torch.from_numpy(cat["latents"]), torch.from_numpy(cat["sizes"]))
    got = c.retrieve(torch.from_numpy(cat["labels"][:4]).to(dev), torch.from_numpy(cat["latents"][:4]).to(dev),
                     torch.from_numpy(cat["sizes"][:4]).to(dev), mode="objfeats")
    assert got.cpu().tolist() == [0, 1, 2, 3]
