"""Shape auto-encoder golden vectors: the UNMODIFIED reference `KLAutoEncoder` (foldingnet_autoencoder.py:337-390) run on
CPU / fp32 with seeded weights.

Run in the authoring container only (needs the reference checkout):
    python tests/golden/make_golden_shape_ae.py
The reference imports the CUDA Chamfer extension (ChamferDistancePytorch/chamfer3D), which is JIT-built and cannot be
built without a GPU; a stand-in module whose chamfer_3DDist calls the reference's own pure-torch
ChamferDistancePytorch/chamfer_python.distChamfer is registered before the import.  Writes tests/golden/sae_*.npz: the
state-dict key list, the points, the eps draws and the three kNN stages' indices (the module-level `knn` wrapped), the
latent, kl, recon, Chamfer distances and indices, get_loss and its dict (train cases), the running statistics after
the pass, and the gradient of every parameter (in full below FULL_GRAD_MAX elements, else norm and a dot product with a seeded probe).
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_golden_class import Recorder   # noqa: E402  (also puts the reference on sys.path)
from tests.cases_shape_ae import FULL_GRAD_MAX, SAE_CASES, probe, sae_points, sae_state_dict  # noqa: E402


def _chamfer_stand_in():
    from ChamferDistancePytorch.chamfer_python import distChamfer

    class chamfer_3DDist(torch.nn.Module):
        def forward(self, a, b):
            return distChamfer(a, b)

    for name in ("ChamferDistancePytorch.chamfer3D", "ChamferDistancePytorch.chamfer3D.dist_chamfer_3D"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["ChamferDistancePytorch.chamfer3D.dist_chamfer_3D"].chamfer_3DDist = chamfer_3DDist


def main():
    _chamfer_stand_in()
    import scene_synthesis.networks.foldingnet_autoencoder as M
    for name, case in SAE_CASES.items():
        net = M.KLAutoEncoder(latent_dim=case["latent_dim"], kl_weight=case["kl_weight"])
        net.load_state_dict(sae_state_dict(net.state_dict(), case), strict=True)
        net.train(case["train"])
        out = {"keys": np.array(list(net.state_dict().keys()))}
        pts = sae_points(case)
        out["points"] = pts.numpy()
        knns, seen = [], {}
        real_knn, real_fwd = M.knn, net.forward
        M.knn = lambda x, k: knns.append(real_knn(x, k)) or knns[-1]

        def forward(pc):
            seen["kl"], seen["lat"], seen["rec"] = real_fwd(pc)
            return seen["kl"], seen["lat"], seen["rec"]
        net.forward = forward
        try:
            with Recorder(case["seed"] + 1) as r:
                if case["train"]:
                    loss, ld = net.get_loss({"points": pts})
                else:
                    with torch.no_grad():
                        net(pts)
        finally:
            M.knn = real_knn
        out["eps"] = r.randn_draws[0].numpy()
        out["knn"] = torch.stack(knns).numpy().astype(np.int16)
        rec = seen["rec"].detach()
        out["latent"], out["kl"], out["recon"] = seen["lat"].detach().numpy(), seen["kl"].detach().numpy(), rec.numpy()
        d1, d2, i1, i2 = M.cd_loss(pts, rec)
        out["dist1"], out["dist2"], out["idx1"], out["idx2"] = d1.numpy(), d2.numpy(), i1.numpy(), i2.numpy()
        for k, v in net.state_dict().items():
            if "running" in k:
                out["rs1." + k] = v.numpy().copy()
        if case["train"]:
            loss.backward()
            out["loss"] = np.asarray(loss.detach().numpy())
            for k, v in ld.items():
                out["ld." + k] = np.asarray(v.detach().numpy())
            for k, p in net.named_parameters():
                g = p.grad.detach()
                out["gnorm." + k] = np.asarray(g.norm().item(), np.float64)
                out["gdot." + k] = np.asarray((g.double() * probe(k, g.shape).double()).sum().item(), np.float64)
                if g.numel() < FULL_GRAD_MAX:
                    out["grad." + k] = g.numpy()
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        print(name, len(out["keys"]), "keys;", {k: getattr(v, "shape", None) for k, v in out.items()
                                                if not k.startswith(("gnorm", "gdot", "grad", "rs"))})


if __name__ == "__main__":
    main()
