"""3-D reconstruction metrics of a finished run, as metric/eval_3D_obj.py and eval_3D_scene.py compute them, on the GPU.

  python tools/eval_3d.py --mode obj   --mesh-dir LOG/scene_mesh --gt-dir DATA/room_0/habitat --out LOG/eval_mesh
  python tools/eval_3d.py --mode scene --mesh-dir LOG/scene_mesh --gt-dir DATA/room_0/habitat --out LOG/eval_mesh

obj:   every frame_{F}_obj{id}.obj in --mesh-dir is scored against mesh_semantic.ply_{id}.ply (id 0: the concatenation of
       the GT meshes whose class is a background class, from info_semantic.json) with 10 000 samples (200 000 for id 0),
       cropped to the GT's enlarged oriented box; writes metric_obj{id}.npy and metrics_3D_obj.npy.
scene: frame_{F}_scene.obj, or else every .obj / .ply of --mesh-dir concatenated, against --gt-dir/../mesh.ply with
       200 000 samples; writes metrics_3D_scene.npy.
Both print the mean ``Acc | Comp | Comp Ratio 1cm | Comp Ratio 5cm`` line.  The arithmetic is vmap_b200.metrics.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from vmap_b200 import metrics  # noqa: E402


def gt_bg_mesh(gt_dir, background_cls):
    with open(os.path.join(gt_dir, "info_semantic.json")) as f:
        objects = json.load(f)["objects"]
    return metrics.concatenate([metrics.load_mesh(os.path.join(gt_dir, "mesh_semantic.ply_%d.ply" % int(o["id"])))
                                for o in objects if int(o["class_id"]) in background_cls])


def eval_obj(a):
    metrics_3d = [[] for _ in range(4)]
    for obj_id in metrics.frame_obj_ids(a.mesh_dir, a.frame):
        if obj_id == 0:
            N, mesh_gt = 200000, gt_bg_mesh(a.gt_dir, a.background_cls)
        else:
            N, mesh_gt = 10000, metrics.load_mesh(os.path.join(a.gt_dir, "mesh_semantic.ply_%d.ply" % obj_id))
        mesh_rec = metrics.load_mesh(os.path.join(a.mesh_dir, "frame_%d_obj%d.obj" % (a.frame, obj_id)))
        m = metrics.calc_3d_metric(mesh_rec, mesh_gt, N=N, crop_to_gt_box=True, seed=a.seed)
        if m is None:
            continue
        np.save(os.path.join(a.out, "metric_obj%d.npy" % obj_id), np.array(m))
        for k in range(4):
            metrics_3d[k].append(m[k])
    metrics_3d = np.array(metrics_3d)
    np.save(os.path.join(a.out, "metrics_3D_obj.npy"), metrics_3d)
    print("metrics 3D obj \n Acc | Comp | Comp Ratio 1cm | Comp Ratio 5cm \n", metrics_3d.mean(axis=1))


def eval_scene(a):
    scene = os.path.join(a.mesh_dir, "frame_%d_scene.obj" % a.frame)
    if os.path.isfile(scene):
        mesh_rec = metrics.load_mesh(scene)
    else:
        mesh_rec = metrics.concatenate([metrics.load_mesh(os.path.join(a.mesh_dir, f)) for f in sorted(os.listdir(a.mesh_dir))
                                        if os.path.splitext(f)[1] in (".obj", ".ply")])
    mesh_gt = metrics.load_mesh(os.path.join(a.gt_dir, "..", "mesh.ply"))
    m = metrics.calc_3d_metric(mesh_rec, mesh_gt, N=200000, seed=a.seed)
    metrics_3d = np.array([[m[k]] for k in range(4)])
    np.save(os.path.join(a.out, "metrics_3D_scene.npy"), metrics_3d)
    print("metrics 3D scene \n Acc | Comp | Comp Ratio 1cm | Comp Ratio 5cm \n ", metrics_3d.mean(axis=1))


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--mesh-dir", required=True, help="the run's scene_mesh directory (frame_{F}_obj{id}.obj)")
    p.add_argument("--gt-dir", required=True, help="the sequence's habitat directory (mesh_semantic.ply_{id}.ply)")
    p.add_argument("--out", required=True, help="output directory for the .npy files")
    p.add_argument("--mode", choices=("obj", "scene"), default="obj")
    p.add_argument("--frame", type=int, default=1999)
    p.add_argument("--background-cls", type=int, nargs="*", default=metrics.BACKGROUND_CLS)
    p.add_argument("--seed", type=int, default=0)
    a = p.parse_args(argv)
    os.makedirs(a.out, exist_ok=True)
    (eval_obj if a.mode == "obj" else eval_scene)(a)


if __name__ == "__main__":
    main()
