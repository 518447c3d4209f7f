"""Host-side timing of the motion detector with its cluster lists (diagnostic; run on a GPU box): per frame,
kb_detect_motion + kb_get_motion_clusters, and kb_spin_once + kb_get_motion_clusters, on 640x480 frames of the dynamic
workload (room scene, slow orbit, a box ~2.2 m in front of the camera covering ~20 % of the pixels, as in
bench.py --workload dynamic). Each sequence runs on frames without a vertex map, with a host vertex map and with a
device-resident vertex map (kb_compute_vertex_map of the frame). The calls are synchronous, so perf_counter around
them is the latency a caller of the Python binding sees. Prints the card and its power limit with the results."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import khronos_b200 as kb
from khronos_b200 import capi, synthetic as syn

BURN = 90       # frames of kb_spin_once before timing: the box appears after 60 frames and the space behind it is ever-free
WARM = 5        # timed-sequence frames left out of the statistics


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name(0)
    return q


def make_handle(cam):
    mc = capi.default_map_config(voxel_size=0.05, vps=16, trunc=0.15, max_blocks=45000)
    ic = capi.default_integrator_config(semantic_mode=capi.SEM_MLE, num_labels=20)
    mot = capi.default_motion_config(min_cluster_size=500, min_separation_distance=2.0)
    h = kb.create_map(mc, ic, capi.default_tracking_config(), mot, device=0)
    h.set_camera(cam)
    return h


def stats(us):
    us = np.asarray(us[WARM:], np.float64)
    return {"mean_us": round(float(us.mean()), 1), "median_us": round(float(np.median(us)), 1),
            "p90_us": round(float(np.percentile(us, 90)), 1)}


def main(n_timed=60):
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    cam = syn.make_camera()
    n = BURN + n_timed
    poses, stamps = syn.orbit_trajectory(n, laps=n / 3000.0)
    depth, label = syn.render_stream(syn.room_scene(20), cam, poses, stamps, device=dev, dtype=torch.float32,
                                     extra=syn.companion_cuboids(poses))
    timed = range(BURN, n)
    # vertex maps of the timed frames (the back-projection, as hydra's createData builds them)
    h = make_handle(cam)
    vdev = torch.empty((n_timed, cam.height, cam.width, 3), dtype=torch.float32, device=dev)
    for k, i in enumerate(timed):
        h.compute_vertex_map(h.make_frame(depth[i].data_ptr(), poses[i], stamps[i], memory=capi.MEM_DEVICE), vdev[k].data_ptr())
    torch.cuda.synchronize()
    vhost = vdev.cpu().numpy()
    dhost, lhost = depth[BURN:].cpu().numpy(), label[BURN:].cpu().numpy()
    del h

    def frame(h, mode, i, with_label):
        k = i - BURN
        if mode == "host_vertex":
            return h.make_frame(dhost[k], poses[i], stamps[i], label=lhost[k] if with_label else None, vertex_world=vhost[k])
        v = vdev[k].data_ptr() if mode == "device_vertex" else None
        return h.make_frame(depth[i].data_ptr(), poses[i], stamps[i], label=label[i].data_ptr() if with_label else None,
                            vertex_world=v, memory=capi.MEM_DEVICE)

    out = {"card": card(), "image": [cam.width, cam.height], "timed_frames": n_timed - WARM}
    for mode in ("no_vertex", "host_vertex", "device_vertex"):
        h = make_handle(cam)
        for i in range(BURN):
            h.spin_once(h.make_frame(depth[i].data_ptr(), poses[i], stamps[i], label=label[i].data_ptr(), memory=capi.MEM_DEVICE),
                        want_image=False)
        h.synchronize()
        res = {}
        for seq in ("detect", "spin_once"):
            us, clusters, pixels = [], 0, 0
            for i in timed:
                f = frame(h, mode, i, seq == "spin_once")
                t0 = time.perf_counter()
                if seq == "detect":
                    _, _, nc = h.detect_motion(f)
                else:
                    _, _, nc = h.spin_once(f)
                cl = h.get_motion_clusters() if nc else []
                us.append((time.perf_counter() - t0) * 1e6)
                clusters += len(cl)
                pixels += sum(len(c["pixels"]) for c in cl)
            res[seq] = dict(stats(us), clusters_per_frame=round(clusters / n_timed, 2), list_pixels_per_frame=round(pixels / n_timed))
        out[mode] = res
        del h
    print(out)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 60)
