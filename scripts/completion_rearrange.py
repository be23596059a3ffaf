#!/usr/bin/env python
"""Scene completion and rearrangement of real scenes (reference scripts/completion_rearrange.py), batched.

    python scripts/completion_rearrange.py CONFIG OUT ROOM_DIR --weight_file W --catalogue catalogue.npz \
        --mesh_catalogue mesh_catalogue.npz [--arrange_objects] [--num_partial 3] [--batch_size 64] ...

ROOM_DIR holds the reference's preprocessed scenes (<room>/boxes.npz, as scripts/render_scenes.py reads them, plus
`room_layout` for floor-plan configs).  Rooms are taken in sorted order.  Each sequence i picks a room as the
reference does (:290-297): room i mod n_rooms when arranging, np.random.choice(n_rooms) after np.random.seed(--seed)
when completing, drawn up front for all sequences; --scene_id (a room directory name) fixes the room.  The scene is
encoded into network space (collate + encode_batch, padded to N rows with the empty class, file order kept) and

  * completion: the first --num_partial rows (padding rows included when the scene is smaller, as in the reference)
    are the partial scene, completed by network.sample(partial_boxes=...);
  * arrangement (--arrange_objects, a config with room_arrange_condition): the reference's noise (:309-324) is added
    in network space -- translations += randn(N, 3) after np.random.seed(scene_idx), or with --scene_id x and z
    replaced by 0.4 randn; angles += randn(N, angle_dim) after np.random.seed(scene_idx + n_rooms) -- and the
    network resamples translations and angles with network.sample(input_boxes=...).

--batch_size sequences are sampled per call, seeded as generate_diffusion.py seeds its batches.  Outputs:
OUT/scene_XXXXX.npz (generate_diffusion.py's layout plus `room`, `scene_idx` and, when rendering, `model_index`), so
`render_scenes.py ROOM_DIR --generated OUT --fid --ipr` scores the results against the real scenes; with
--mesh_catalogue, renders of the input (OUT/partial or OUT/noisy/<room>_<idx>_<i:03d>_render.png), of the result
(OUT/<room>_<idx>_<i:03d>.png) and, with --gen_gt, of the real scene (OUT/groundtruth/...), every one placed with the
models --catalogue retrieves.  The camera is the reference's perspective view (diffuscene_b200.render.
REFERENCE_PERSPECTIVE, or --camera_position / --camera_target / --up_vector / --window_size) on a white background,
or the top-down camera with --render_top2down.  The shading is this project's, not simple-3dviz's.
--compute_intersec appends generate_diffusion.py's iou_states.txt lines.
"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from training_utils import load_config  # noqa: E402

from diffuscene_b200.collate import collate_scenes  # noqa: E402
from diffuscene_b200.postprocess import encode_batch, load_dataset_stats, post_process_batch  # noqa: E402
from diffuscene_b200.synthetic import DEFAULT_BOUNDS  # noqa: E402


def _floats(x):
    return tuple(float(v) for v in x.split(","))


def parse_args(argv):
    p = argparse.ArgumentParser(description="Complete or rearrange real scenes with a trained model")
    p.add_argument("config_file")
    p.add_argument("output_directory")
    p.add_argument("room_dir", help="directory of <room>/boxes.npz (the reference's preprocessed scenes)")
    p.add_argument("--weight_file", default=None)
    p.add_argument("--dataset_stats", default=None,
                   help="the reference's dataset_stats.txt (default: the synthetic bounds generate_diffusion.py uses)")
    p.add_argument("--n_sequences", default=10, type=int)
    p.add_argument("--batch_size", default=64, type=int, help="sequences sampled per call")
    p.add_argument("--num_partial", default=3, type=int)
    p.add_argument("--arrange_objects", action="store_true")
    p.add_argument("--scene_id", default=None, help="room directory name to use for every sequence")
    p.add_argument("--clip_denoised", action="store_true")
    p.add_argument("--ddim", action="store_true")
    p.add_argument("--ddim_steps", type=int, default=50)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    p.add_argument("--gen_gt", action="store_true", help="also render the real scenes (or validation.gen_gt)")
    p.add_argument("--compute_intersec", action="store_true", help="append scene statistics to iou_states.txt")
    p.add_argument("--catalogue", default=None, help="catalogue.npz of the models to place (default: boxes)")
    p.add_argument("--retrieve_mode", default=None, choices=["objfeats", "objfeats_and_size", "box"])
    p.add_argument("--mesh_catalogue", default=None, help="mesh_catalogue.npz: render inputs and results")
    p.add_argument("--render_top2down", action="store_true", help="top-down renders instead of the perspective view")
    p.add_argument("--no_texture", action="store_true")
    p.add_argument("--without_floor", action="store_true")
    p.add_argument("--floor_textures", default=None, help="folder of floor textures (default: a white floor)")
    p.add_argument("--window_size", type=lambda x: tuple(int(v) for v in x.split(",")), default=(512, 512))
    p.add_argument("--camera_position", type=_floats, default=(-0.10923499, 1.9325259, -7.19009))
    p.add_argument("--camera_target", type=_floats, default=(0.0, 0.0, 0.0))
    p.add_argument("--up_vector", type=_floats, default=(0.0, 1.0, 0.0))
    args = p.parse_args(argv)
    if args.n_sequences < 1 or args.batch_size < 1:
        p.error("--n_sequences and --batch_size must be >= 1")
    if args.mesh_catalogue is not None and args.catalogue is None:
        p.error("--mesh_catalogue needs the --catalogue that retrieves from it")
    if len(args.window_size) != 2 or min(args.window_size) < 1 or max(args.window_size) > 4096:
        p.error("--window_size must be W,H in [1, 4096]")
    for name in ("camera_position", "camera_target", "up_vector"):
        if len(getattr(args, name)) != 3:
            p.error("--%s needs three comma-separated numbers" % name)
    config = load_config(args.config_file)
    net = config["network"]
    N = int(net["sample_num_points"])
    if args.arrange_objects and not net.get("room_arrange_condition", False):
        p.error("--arrange_objects needs a config with room_arrange_condition (config/rearrange)")
    if not args.arrange_objects and not 1 <= args.num_partial <= N:
        p.error("--num_partial must lie in [1, %d]" % N)
    if not os.path.isdir(args.room_dir):
        p.error("no room directory %s" % args.room_dir)
    return args, config


def choose_scenes(n_sequences, n_rooms, arrange, scene_idx=None, seed=0):
    """Room index of every sequence (reference :290-297) after np.random.seed(seed); `scene_idx` fixes the room."""
    np.random.seed(seed)
    out = []
    for i in range(n_sequences):
        if arrange:
            idx = scene_idx if scene_idx is not None else i % n_rooms
        else:
            idx = scene_idx if scene_idx is not None else int(np.random.choice(n_rooms))
        out.append(idx)
    return out


def arrangement_noise(scene_indices, n_rooms, N, angle_dim, fixed_scene):
    """The reference's arrangement noise per sequence (:309-324), in its call order: (translation noise [N, 3],
    replace x and z instead of adding, angle noise [N, angle_dim])."""
    out = []
    for idx in scene_indices:
        if fixed_scene:
            nt = 0.4 * np.random.randn(N, 3).astype(np.float32)
        else:
            np.random.seed(idx)
            nt = np.random.randn(N, 3).astype(np.float32)
        np.random.seed(idx + n_rooms)
        na = np.random.randn(N, angle_dim).astype(np.float32)
        out.append((nt, fixed_scene, na))
    return out


def encode_scenes(scenes, N, bounds, objfeat_dim=0, objectness_dim=0):
    """Network-space rows [B, N, d] of real scenes: translations, sizes, angles (cos, sin), class labels in {-1, +1}
    with the end label on padding rows, [objectness], [objfeats]; padding rows are zero elsewhere."""
    rows = []
    fkey = "objfeats_32" if objfeat_dim == 32 else "objfeats"
    for s in scenes:
        L = len(s["class_labels"])
        world = {k: torch.as_tensor(np.asarray(s[k], np.float32).reshape(L, -1)) for k in ("translations", "sizes")}
        world["angles"] = torch.as_tensor(np.asarray(s["angles"], np.float32).reshape(L, 1))
        if objfeat_dim > 0:
            f = s.get(fkey, s.get("objfeats"))
            world["objfeats_32" if fkey == "objfeats_32" else "objfeats"] = torch.as_tensor(
                np.zeros((L, objfeat_dim), np.float32) if f is None else np.asarray(f, np.float32).reshape(L, -1))
        b = dict(bounds)
        if objfeat_dim > 0 and fkey not in b:
            b[fkey] = b.get("objfeats", b.get("objfeats_32"))
        enc = encode_batch(world, b)
        enc["class_labels"] = np.asarray(s["class_labels"], np.float32)
        rows.append(enc)
    batch = collate_scenes(rows, N)
    parts = [batch["translations"], batch["sizes"], batch["angles"], batch["class_labels"]]
    if objectness_dim > 0:
        real = (torch.arange(N)[None] < batch["length"][:, None]).float()[..., None]
        parts.append(1 - 2 * real)
    if objfeat_dim > 0:
        parts.append(batch[fkey])
    return torch.cat(parts, dim=-1)


def room_layout(s, size):
    """The reference's room mask (threed_front.py:311-319): room_layout[:, :, 0] resized with PIL bilinear, / 255."""
    from PIL import Image
    img = Image.fromarray(np.asarray(s["room_layout"])[:, :, 0])
    img = img.resize(size, resample=Image.BILINEAR)
    return np.asarray(img).astype(np.float32) / np.float32(255)


def main(argv):
    args, config = parse_args(argv)
    from render_scenes import load_rooms
    rooms, raw = load_rooms(args.room_dir)
    fixed = None
    if args.scene_id is not None:
        if args.scene_id not in rooms:
            raise SystemExit("--scene_id %s is not a room under %s" % (args.scene_id, args.room_dir))
        fixed = rooms.index(args.scene_id)
    bounds = load_dataset_stats(args.dataset_stats) if args.dataset_stats else DEFAULT_BOUNDS
    gen_gt = args.gen_gt or bool(config.get("validation", {}).get("gen_gt", False))
    if not torch.cuda.is_available():
        raise RuntimeError("completion_rearrange.py needs a CUDA device (H100); there is no CPU path")

    from scene_synthesis.networks import build_network
    from diffuscene_b200.evaluate import PlausibilityAggregator, evaluate_samples, place_samples
    from diffuscene_b200.synthetic import SyntheticScenes
    from generate_diffusion import _catalogue
    device = torch.device("cuda:0")
    os.makedirs(args.output_directory, exist_ok=True)
    torch.manual_seed(args.seed)
    config["network"]["diffusion_kwargs"]["loss_iou"] = False
    ds = SyntheticScenes(config["network"], 1)
    network, _, _ = build_network(ds.feature_size, ds.n_classes, config, args.weight_file, device=device,
                                  precision=args.precision)
    network.eval()
    N, d = config["network"]["sample_num_points"], config["network"]["point_dim"]
    angle_dim = network.bbox_dim - network.translation_dim - network.size_dim

    # inputs of every sequence, drawn up front in the reference's order
    order = choose_scenes(args.n_sequences, len(rooms), args.arrange_objects, fixed, args.seed)
    x_real = encode_scenes(raw, N, bounds, network.objfeat_dim, network.objectness_dim)     # [n_rooms, N, d]
    if x_real.shape[-1] != d:
        raise ValueError("encoded scenes have %d channels, the network %d" % (x_real.shape[-1], d))
    x_in = x_real[order].clone()
    if args.arrange_objects:
        td, sd = network.translation_dim, network.size_dim
        for i, (nt, replace, na) in enumerate(arrangement_noise(order, len(rooms), N, angle_dim, fixed is not None)):
            if replace:
                x_in[i, :, 0] = torch.from_numpy(nt[:, 0])
                x_in[i, :, 2] = torch.from_numpy(nt[:, 2])
            else:
                x_in[i, :, :td] += torch.from_numpy(nt)
            x_in[i, :, td + sd:td + sd + angle_dim] += torch.from_numpy(na)
        folder = "noisy"
    else:
        x_in = x_in[:, :args.num_partial].contiguous()
        folder = "partial"
    if network.room_mask_condition:
        size = tuple(int(v) for v in str(config.get("data", {}).get("room_layout_size", "64,64")).split(","))
        masks = torch.from_numpy(np.stack([room_layout(s, size) for s in raw]))[:, None]
    names = ["{}_{}_{:03d}".format(rooms[idx], idx, i) for i, idx in enumerate(order)]

    if args.compute_intersec:
        catalog, mode = _catalogue(args.catalogue, network, args.retrieve_mode)
        aggs, modes = [PlausibilityAggregator(PlausibilityAggregator.SUFFIX_OBJFEATS)], [mode]
        if catalog is not None and mode != "box":
            aggs.append(PlausibilityAggregator(PlausibilityAggregator.SUFFIX_ONLYSIZE))
            modes.append("box")
    render = args.mesh_catalogue is not None
    if render:
        from PIL import Image
        from diffuscene_b200 import render as R
        render_cat, render_mode = _catalogue(args.catalogue, network, args.retrieve_mode)
        meshes = R.MeshCatalog(args.mesh_catalogue)
        if meshes.num_models != len(render_cat.model_ids):
            raise ValueError("the mesh catalogue holds %d models, the retrieval catalogue %d"
                             % (meshes.num_models, len(render_cat.model_ids)))
        palette = R.hls_palette(network.class_dim - 1)
        if args.render_top2down:
            camera, white = R.Camera(), args.without_floor
        else:
            W, H = args.window_size
            camera = R.Camera.perspective(args.camera_position, args.camera_target, args.up_vector, width=W, height=H)
            white = True
        floor_tex = R.load_floor_textures(args.floor_textures) if args.floor_textures else None
        for sub in (folder, "groundtruth") if gen_gt else (folder,):
            os.makedirs(os.path.join(args.output_directory, sub), exist_ok=True)

        def draw(rows, scene_ids, seed):
            """Renders of network-space rows [b, n, d] of the rooms `scene_ids`, placed with retrieved models."""
            world, keep, cls, mi = place_samples(network, rows.to(device), bounds, render_cat, render_mode)
            mi = torch.where(keep, mi, -1)
            floors = None if args.without_floor else R.floor_triangles(
                [(raw[j]["floor_plan_vertices"] - raw[j]["floor_plan_centroid"], raw[j]["floor_plan_faces"])
                 if "floor_plan_vertices" in raw[j] else None for j in scene_ids])
            fti = None
            if floor_tex is not None and floors is not None:
                fti = R.choose_floor_textures(len(scene_ids), len(floor_tex), seed)
            img = R.render_scenes(meshes, world["translations"], world["sizes"], world["angles"], mi, cls,
                                  floors=floors, no_texture=args.no_texture, white_background=white, camera=camera,
                                  palette=palette, floor_textures=floor_tex, floor_texture_index=fti)
            return img.cpu().numpy(), mi

    done = 0
    while done < args.n_sequences:
        bs = min(args.batch_size, args.n_sequences - done)
        sl = slice(done, done + bs)
        ids = order[sl]
        room_mask = masks[ids].to(device) if network.room_mask_condition else torch.zeros(bs, 1, 64, 64, device=device)
        kw = dict(batch_size=bs, clip_denoised=args.clip_denoised, ddim=args.ddim, ddim_steps=args.ddim_steps,
                  seed=args.seed * 100003 + done)
        if args.arrange_objects:
            samples = network.sample(room_mask, N, d, input_boxes=x_in[sl].to(device), **kw)
        else:
            samples = network.sample(room_mask, N, d, partial_boxes=x_in[sl].to(device), **kw)
        if render:
            seed = args.seed + done
            inp, _ = draw(x_in[sl], ids, seed)
            res, mi = draw(samples, ids, seed)
            kept_models = [mi[b][~(samples[b, :, network.bbox_dim + network.class_dim - 1] >= 0)].cpu().numpy()
                           for b in range(bs)]
            gt = draw(x_real[ids], ids, seed)[0] if gen_gt else None
            for b in range(bs):
                name = names[done + b]
                Image.fromarray(inp[b]).save(os.path.join(args.output_directory, folder, name + "_render.png"))
                Image.fromarray(res[b]).save(os.path.join(args.output_directory, name + ".png"))
                if gt is not None:
                    Image.fromarray(gt[b]).save(os.path.join(args.output_directory, "groundtruth",
                                                             name + "_render.png"))
        for b, scene in enumerate(network.delete_empty_batched(samples)):
            boxes = {k: v[None] for k, v in scene.items() if k != "class_index"}
            pb = dict(bounds)
            if "objfeats" in boxes and "objfeats" not in pb:
                pb["objfeats"] = pb.get("objfeats_32", DEFAULT_BOUNDS["objfeats_32"])
            out = {k: v.numpy() for k, v in post_process_batch(boxes, pb).items()}
            out["class_index"] = scene["class_index"].numpy()
            out["room"], out["scene_idx"] = np.array(rooms[ids[b]]), np.array(ids[b])
            if render:
                out["model_index"] = kept_models[b]
            np.savez(os.path.join(args.output_directory, "scene_{:05d}.npz".format(done + b)), **out)
        if args.compute_intersec:
            lines = [agg.update(evaluate_samples(network, samples, bounds, catalog, m)) for agg, m in zip(aggs, modes)]
            with open(os.path.join(args.output_directory, "iou_states.txt"), "a") as f:
                for per_scene in zip(*lines):
                    f.write("".join(line + "\n" for line in per_scene))
        done += bs
    print("{} {} scenes into {}".format("arranged" if args.arrange_objects else "completed", done,
                                        args.output_directory))


if __name__ == "__main__":
    main(sys.argv[1:])
