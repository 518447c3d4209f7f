"""kb_generate_mesh against the from-spec model (mesh_model.py) run on the product's own export, and bit for bit against the
oracle: the scenes of test_mesh_model.py, block counts around the single-CTA scan's 1024-thread boundary, one handle across
growing and empty calls, in-process sharded handles (whose border cubes are dropped), and the benchmark's hall640 map."""
import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import harness as hs
import mesh_model as mm
from test_mesh_oracle import TABLE
from test_mesh_model import (CASES, OFFSETS, SCENES, SCENE_TARGETS, VS, again_fn, assert_mesh_equals_model, check_handle, flat,
                             labels_image, pose, stamp, voxel_size_of, _handle)
from test_zz_mesh import assert_mesh_equal

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("vps", [8, 16])
@pytest.mark.parametrize("name,offname", CASES)
def test_product_mesh_equals_model_and_oracle(oracle_lib, product_lib, name, offname, vps):
    off = OFFSETS[offname]
    meshes, infos = {}, {}
    for lib, prefix in ((oracle_lib, "ko_"), (product_lib, "kb_")):
        h, info = SCENES[name](lib, prefix, vps, off)
        meshes[prefix], counts, missing, _ = check_handle(h, voxel_size_of(name), vps, f"{prefix}{name}/{offname}/vps{vps}",
                                                          again=again_fn(name, off))
        assert SCENE_TARGETS[name](counts, info, missing), (prefix, name, counts)
        infos[prefix] = info
    assert infos["ko_"].keys() == infos["kb_"].keys() and all(infos["ko_"][k] == infos["kb_"][k] for k in infos["ko_"])
    assert len(meshes["ko_"]) == len(meshes["kb_"])
    for k, (mo, mg) in enumerate(zip(meshes["ko_"], meshes["kb_"])):
        assert_mesh_equal(mo, mg, f"{name}/{offname}/vps{vps} call {k}")


@pytest.mark.parametrize("vps", [8, 16])
def test_removal_after_rehash(oracle_lib, product_lib, monkeypatch, vps):
    """The removal scene with the hash rebuilt after every removal, so that the survivors' missing neighbours are looked
    up in a freshly rebuilt table rather than past tombstones."""
    monkeypatch.setenv("KB_REHASH_TOMBSTONES", "1")
    g, info = SCENES["removal"](product_lib, "kb_", vps, OFFSETS["origin"])
    o, info_o = SCENES["removal"](oracle_lib, "ko_", vps, OFFSETS["origin"])
    assert info["removed"] == info_o["removed"] and info["removed"]
    mg, counts, missing, _ = check_handle(g, VS, vps, "rehash", again=again_fn("removal", OFFSETS["origin"]))
    mo, *_ = check_handle(o, VS, vps, "rehash oracle", again=again_fn("removal", OFFSETS["origin"]))
    assert missing & info["removed"]
    for k, (a, b) in enumerate(zip(mo, mg)):
        assert_mesh_equal(a, b, f"rehash call {k}")


def _box_map(lib, prefix, boxes, vps=8):
    """Blocks allocated as the given boxes, fused with allocate_blocks = False from a camera looking into them."""
    h = _handle(lib, prefix, vps, map_kw={"max_blocks": 4096})
    for lo, hi in boxes:
        h.allocate_box(lo, hi)
    d = flat(2.0 + VS / 2)
    h.integrate_frame(h.make_frame(d, pose((0.0, 0.0, 0.0)), stamp(0), label=labels_image()), allocate_blocks=False)
    return h


# 0.5 m blocks: x in [2, 10), y, z around the camera axis; 1024 = 16 x 8 x 8, 1025 = that + one, 2304 = 16 x 12 x 12
BOX_SETS = {1024: [((2, -4, -4), (17, 3, 3))],
            1025: [((2, -4, -4), (17, 3, 3)), ((18, 0, 0), (18, 0, 0))],
            2304: [((2, -6, -6), (17, 5, 5))]}


@pytest.mark.parametrize("n_blocks", sorted(BOX_SETS))
def test_block_count_boundaries(oracle_lib, product_lib, n_blocks):
    o = _box_map(oracle_lib, "ko_", BOX_SETS[n_blocks])
    g = _box_map(product_lib, "kb_", BOX_SETS[n_blocks])
    eg = g.export_blocks(likelihoods=False)
    assert eg.n == n_blocks
    model = mm.mesh(eg, VS, 8, TABLE, only_mesh_updated=False)
    assert model.counts["processed"] == n_blocks and len(model.points) > 1000
    mg = g.generate_mesh(False, False)
    assert_mesh_equals_model(mg, model, f"{n_blocks} blocks")
    assert_mesh_equal(o.generate_mesh(False, False), mg, f"{n_blocks} blocks vs oracle")


def test_one_handle_growing_then_empty(oracle_lib, product_lib):
    """Small map, then a larger one (the block and triangle buffers grow), then a call that processes no block."""
    hs_ = {}
    for lib, prefix in ((oracle_lib, "ko_"), (product_lib, "kb_")):
        h = _handle(lib, prefix, 8, map_kw={"max_blocks": 4096})
        h.allocate_box((3, -1, -1), (4, 0, 0))
        h.integrate_frame(h.make_frame(flat(2.0 + VS / 2), pose((0, 0, 0)), stamp(0), label=labels_image()), allocate_blocks=False)
        hs_[prefix] = h
    seq = []
    for prefix, h in hs_.items():
        out = []
        e = h.export_blocks(likelihoods=False)
        m = h.generate_mesh(True, True)
        assert_mesh_equals_model(m, mm.mesh(e, VS, 8, TABLE, only_mesh_updated=True), f"{prefix} small")
        out.append(m)
        h.allocate_box((2, -6, -6), (17, 5, 5))
        h.integrate_frame(h.make_frame(flat(3.0 + VS / 2), pose((0, 0, 0)), stamp(1), label=labels_image()), allocate_blocks=False)
        e = h.export_blocks(likelihoods=False)
        m = h.generate_mesh(False, True)
        assert_mesh_equals_model(m, mm.mesh(e, VS, 8, TABLE, only_mesh_updated=False), f"{prefix} large")
        assert len(m[0]) == 2304 and len(m[2]) > len(out[0][2])
        out.append(m)
        m = h.generate_mesh(True, True)
        assert len(m[0]) == 0 and m[1].tolist() == [0] and len(m[2]) == 0
        out.append(m)
        out.append(h.generate_mesh(True, False))
        assert len(out[-1][0]) == 0
        seq.append(out)
    for k, (a, b) in enumerate(zip(*seq)):
        assert_mesh_equal(a, b, f"call {k}")


@pytest.mark.parametrize("nranks", [2, 3])
def test_sharded_handles_drop_their_border_cubes(oracle_lib, product_lib, nranks):
    """In-process shards on one device, fed the same frames: each shard's mesh equals the model on that shard's export
    and the oracle's shard, and cubes whose neighbour block lives on another shard are dropped (the documented seams)."""
    cam = hs.small_camera(4)
    poses, stamps = syn.orbit_trajectory(4, laps=0.1)
    rendered = hs.render_frames(syn.room_scene(), cam, poses, stamps)
    mc = capi.default_map_config(vps=8, max_blocks=8192)
    owned = []
    for rank in range(nranks):
        pair = []
        for lib, prefix in ((oracle_lib, "ko_"), (product_lib, "kb_")):
            h = hs.make_handle(lib, prefix, map_cfg=mc, cam=cam)
            h.set_shard(rank, nranks)
            hs.run_fusion(h, rendered, poses, stamps)
            e = h.export_blocks(likelihoods=False)
            model = mm.mesh(e, 0.05, 8, TABLE, only_mesh_updated=False)
            m = h.generate_mesh(False, False)
            assert_mesh_equals_model(m, model, f"{prefix} shard {rank}/{nranks}")
            pair.append((m, model, {tuple(b) for b in e.block_index.tolist()}))
        assert_mesh_equal(pair[0][0], pair[1][0], f"shard {rank}/{nranks} vs oracle")
        owned.append(pair[1])
    everything = set().union(*(own for _, _, own in owned))
    for rank, (_, model, own) in enumerate(owned):
        seams = model.missing & (everything - own)
        assert seams, f"shard {rank}: no border cube was dropped for a block of another shard"


def test_hall640_map_against_model(product_lib):
    """The benchmarked configuration's map (640x480 hall frames, one 32-frame call), meshed with only_mesh_updated=False."""
    import torch
    cam = syn.make_camera()
    poses, stamps = syn.sweep_trajectory(5000)
    poses, stamps = poses[800:832], stamps[800:832]
    d, l = syn.render_stream(syn.hall_scene(20), cam, poses, stamps, device="cuda", dtype=torch.float32)
    d, l = d.cpu().numpy(), l.cpu().numpy()
    g = capi.MapHandle(product_lib, "kb_", capi.default_map_config(max_blocks=8192), capi.default_integrator_config(num_threads=-1),
                       capi.default_tracking_config(), None)
    g.set_camera(cam)
    g.integrate_frames([g.make_frame(d[i], poses[i], stamps[i], label=l[i]) for i in range(32)])
    e = g.export_blocks(likelihoods=False)
    model = mm.mesh(e, 0.05, 16, TABLE, only_mesh_updated=False)
    assert model.counts["processed"] > 300 and len(model.points) > 50000
    assert_mesh_equals_model(g.generate_mesh(False, False), model, "hall640")
