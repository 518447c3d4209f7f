"""Long kb_integrate_frames calls shaped like the benchmark's, against the oracle bit for bit. bench.py makes one
5000-frame call per step on a caller stream with device frames and no stats: 157 pipelined 32-frame batches, whose
prologues (tile pyramid, K0, K0b, K0c) overlap the previous batch's fuse kernel and whose work lists, pyramids, item lists
and counters alternate between two buffer sets by batch parity. Here about 1000 frames of the hall640 stream run in one
call, so that a buffer set is reused while older batches may still be in flight, followed by ragged tails that end in
pipelined batches with and without the item list and in short batches on the main stream, and by a second call that
revisits the same poses (K0 only finds blocks). A seeded fuzzer mixes call lengths with the map operations that order
pipelined prologues behind main-stream work.

Each test derives the host's batch schedule (`Schedule`, a restatement of integrateBatch's splitting and parity
rules) and asserts that it covers what it is meant to: at least three pipelined batches in one call, both parities and a
short batch right after a pipelined one.

Cases that take more than about a minute carry `gpu(slow=True)`; `-m "gpu and not gpu(slow=True)"` leaves them out."""
import functools

import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import harness as hs

pytestmark = pytest.mark.gpu

K_MAX_BATCH = 32
N_LONG, N_REVISIT = 1024 + 19, 32 * 9 + 3
TAILS = (19, 5, 3)   # pipelined with the item list (>= 8 frames), pipelined without it (4-7), short (1-3)


class Schedule:
    """The batches kb_integrate_frames issues, per handle: integrateBatch cuts a call into kMaxBatch-frame batches and
    splits a batch recursively (halves) while the union of its frusta's enumeration boxes exceeds 8 single boxes; every
    (sub-)batch flips the handle's parity; batches of >= 4 frames are pipelined (KB_PIPELINE on)."""

    def __init__(self, cam, block_size):
        self.cam, self.bs, self.parity = cam, block_size, 0
        self.calls = []   # one list of (n, pipelined, parity) per call

    def _batch(self, poses, allocate, out):
        n = len(poses)
        if allocate and n > 1:
            reach = float(self.cam.max_range) + self.bs * 0.8660254
            t = np.array([np.asarray(T)[:3, 3] for T in poses])
            lo, hi = np.floor((t - reach) / self.bs).min(0), np.floor((t + reach) / self.bs).max(0)
            if not np.prod(hi - lo + 1.0) <= 8.0 * (2.0 * reach / self.bs + 2.0) ** 3:
                self._batch(poses[:n // 2], allocate, out)
                self._batch(poses[n // 2:], allocate, out)
                return
        out.append((n, n >= 4, self.parity))
        self.parity ^= 1

    def call(self, poses, allocate=True):
        out = []
        for i in range(0, len(poses), K_MAX_BATCH):
            self._batch(list(poses[i:i + K_MAX_BATCH]), allocate, out)
        self.calls.append(out)
        return out

    def assert_covers(self):
        """>= 3 pipelined batches in one call, both parities among pipelined batches, a short batch after a pipelined one."""
        assert max(sum(p for _, p, _ in c) for c in self.calls) >= 3, self.calls
        assert {par for c in self.calls for _, p, par in c if p} == {0, 1}, self.calls
        flat = [p for c in self.calls for _, p, _ in c]
        assert any(a and not b for a, b in zip(flat, flat[1:])), self.calls


def hall_cfg():
    """bench.py's hall640 map: 5 cm voxels, 16^3 blocks, tracking layer, MLE with L = 20, default culling."""
    mc = capi.default_map_config(voxel_size=0.05, vps=16, trunc=0.15, with_semantics=True, with_tracking=True, max_blocks=45000)
    ic = capi.default_integrator_config(semantic_mode=capi.SEM_MLE, num_labels=20, num_threads=-1)
    return mc, ic


@functools.lru_cache(maxsize=1)
def hall_stream():
    """hall640 frames 0..N_LONG of the 5000-frame lap, rendered on the GPU and kept there, plus the revisit: the first
    N_REVISIT poses again with later stamps."""
    import torch
    cam = syn.make_camera()
    poses, stamps = syn.sweep_trajectory(5000)
    poses, stamps = poses[:N_LONG], stamps[:N_LONG]
    d, l = syn.render_stream(syn.hall_scene(20), cam, poses, stamps, device="cuda", dtype=torch.float32)
    rev_stamps = [stamps[-1] + (i + 1) * 33_333_333 for i in range(N_REVISIT)]
    torch.cuda.synchronize()
    return cam, poses, stamps, d, l, poses[:N_REVISIT], rev_stamps


@functools.lru_cache(maxsize=1)
def _oracle_result(oracle_path):
    import ctypes
    cam, poses, stamps, d, l, rposes, rstamps = hall_stream()
    mc, ic = hall_cfg()
    o = capi.MapHandle(ctypes.CDLL(oracle_path), "ko_", mc, ic, capi.default_tracking_config(), None)
    o.set_camera(cam)

    def feed(ps, sts, src):   # 32 frames at a time from the GPU tensors: never the whole stream on the host twice
        for b0 in range(0, len(ps), K_MAX_BATCH):
            idx = list(range(b0, min(b0 + K_MAX_BATCH, len(ps))))
            dh, lh = d[src[0]:src[1]][idx].cpu().numpy(), l[src[0]:src[1]][idx].cpu().numpy()
            o.integrate_frames([o.make_frame(dh[k], ps[i], sts[i], label=lh[k]) for k, i in enumerate(idx)], want_stats=False)
    feed(poses, stamps, (0, N_LONG))
    feed(rposes, rstamps, (0, N_REVISIT))
    t = o.get_totals64().as_dict()
    return o.export_blocks(), o.map_checksum(), t


@pytest.fixture(scope="module")
def hall_oracle(oracle_lib):
    """The oracle's map after the long stream and the revisit: computed once per session, shared by all cases."""
    return _oracle_result(oracle_lib._name)


def run_long_calls(product_lib, tail):
    """The product side: one call of 1024 + tail frames, the rest of the stream in a second call, then the revisit,
    device frames on a caller stream, no stats, no synchronisation until the end."""
    import torch
    cam, poses, stamps, d, l, rposes, rstamps = hall_stream()
    mc, ic = hall_cfg()
    g = capi.MapHandle(product_lib, "kb_", mc, ic, capi.default_tracking_config(), None)
    g.set_camera(cam)
    s = torch.cuda.Stream()
    g.set_stream(s.cuda_stream)
    sched = Schedule(cam, 0.05 * 16)
    cut = 1024 + tail

    def call(lo, hi, ps, sts):
        fr = [g.make_frame(d[i].data_ptr(), ps[i], sts[i], label=l[i].data_ptr(), memory=capi.MEM_DEVICE) for i in range(lo, hi)]
        g.integrate_frames(fr, want_stats=False)
        sched.call(ps[lo:hi])
    call(0, cut, poses, stamps)
    if cut < N_LONG:
        call(cut, N_LONG, poses, stamps)
    call(0, N_REVISIT, rposes, rstamps)
    g.synchronize()
    assert sched.calls[0][-1][0] == tail and sum(n for n, _, _ in sched.calls[0]) == cut
    return g, sched


def assert_matches_oracle(g, oracle, what):
    bo, cs_o, to = oracle
    bg = g.export_blocks()
    hs.assert_blocks_equal(bo, bg, exact_float=True, what=what)
    np.testing.assert_array_equal(bo.semantic_likelihoods.view(np.uint32), bg.semantic_likelihoods.view(np.uint32), err_msg=what)
    cs = g.map_checksum()
    assert cs == cs_o == hs.map_checksum(bg), what
    del bg
    tg = g.get_totals64().as_dict()
    for k in ("blocks_in_frustum", "blocks_allocated", "blocks_updated", "voxels_updated", "voxels_in_band", "voxels_semantic",
              "total_blocks", "capacity_exceeded", "frames"):
        assert tg[k] == to[k], (what, k, tg[k], to[k])
    assert 0 < tg["block_frame_pairs"] < tg["blocks_in_frustum"], what   # culling really ran
    assert tg["frames"] == N_LONG + N_REVISIT and tg["capacity_exceeded"] == 0


@pytest.mark.gpu(slow=True)
@pytest.mark.parametrize("tail", TAILS)
def test_long_pipelined_call_equals_oracle(product_lib, hall_oracle, tail):
    g, sched = run_long_calls(product_lib, tail)
    sched.assert_covers()
    assert sum(p for _, p, _ in sched.calls[0]) >= 32
    assert_matches_oracle(g, hall_oracle, f"long call tail {tail}")


# ---- seeded schedule fuzzer (320x240: four times cheaper for the oracle than hall640, same field of view) ----------------
FUZZ_LENGTHS = (1, 2, 3, 4, 5, 7, 8, 31, 32, 33, 64, 65, 97)


@functools.lru_cache(maxsize=1)
def fuzz_stream(n=900):
    import torch
    cam = syn.make_camera(320, 240, 160.0, 160.0)
    poses, stamps = syn.sweep_trajectory(n, size=(30.0, 20.0), margin=4.0, lanes=3, yaw_turns=6.0)
    d, l = syn.render_stream(syn.hall_scene(20, size=(30.0, 20.0, 6.0)), cam, poses, stamps, device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    return cam, poses, stamps, d, l


@pytest.mark.parametrize("seed,checkpoints", [pytest.param(1, True, marks=pytest.mark.gpu(slow=True)), pytest.param(2, True, marks=pytest.mark.gpu(slow=True)),
                                             (3, False), (4, False)])
def test_schedule_fuzzer_equals_oracle(oracle_lib, product_lib, seed, checkpoints):
    """Random call lengths; between calls, at random: a tracking pass, block removal + clear_updated, a motion detection
    followed by a frame masked with it, host / pinned-async / device frames, stats on or off. One call jumps 400 m in its
    middle, so integrateBatch splits a batch inside a long call. Checkpoint seeds compare the export (which synchronises)
    after some calls; the others compare only at the end, letting every call overlap the next."""
    import torch
    cam, poses, stamps, d, l = fuzz_stream()
    rng = np.random.default_rng(seed)
    mc = capi.default_map_config(voxel_size=0.05, vps=16, trunc=0.15, max_blocks=45000)
    ic = capi.default_integrator_config(num_threads=-1)
    mot = capi.default_motion_config(min_cluster_size=5, min_separation_distance=2.0)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc, integ_cfg=ic, mot_cfg=mot)
    g = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=mc, integ_cfg=ic, mot_cfg=mot)
    s = torch.cuda.Stream()
    g.set_stream(s.cuda_stream)
    sched = Schedule(cam, 0.05 * 16)
    jump = np.eye(4)
    jump[:3, 3] = (400.0, 0.0, 0.0)
    keep = []   # MEM_HOST_ASYNC buffers stay alive (and unchanged) until the next synchronisation
    i, jumped, n = 0, False, len(poses)
    while i < n:
        k = int(min(rng.choice(FUZZ_LENGTHS), n - i))
        ps = [np.asarray(T) for T in poses[i:i + k]]
        if not jumped and k >= 64:
            ps = ps[:k // 2 + 5] + [jump @ T for T in ps[k // 2 + 5:]]   # inside a 32-frame batch
            jumped = True
        mem = rng.choice([capi.MEM_DEVICE, capi.MEM_HOST, capi.MEM_HOST_ASYNC, -1])
        fo, fg = [], []
        for j in range(k):
            dh, lh = d[i + j].cpu().numpy(), l[i + j].cpu().numpy()
            fo.append(o.make_frame(dh, ps[j], stamps[i + j], label=lh))
            m = mem if mem >= 0 else rng.choice([capi.MEM_DEVICE, capi.MEM_HOST])   # -1: mixed within the call
            if m == capi.MEM_DEVICE:
                fg.append(g.make_frame(d[i + j].data_ptr(), ps[j], stamps[i + j], label=l[i + j].data_ptr(), memory=capi.MEM_DEVICE))
            else:
                if m == capi.MEM_HOST_ASYNC:
                    dh, lh = torch.from_numpy(dh).pin_memory(), torch.from_numpy(lh).pin_memory()
                    keep.append((dh, lh))
                fg.append(g.make_frame(dh, ps[j], stamps[i + j], label=lh, memory=int(m)))
        stats = bool(rng.random() < 0.3)
        if stats:
            so = o.integrate_frames(fo).as_dict()
            sg = g.integrate_frames(fg).as_dict()
            assert so == sg, (seed, i, so, sg)
        else:
            o.integrate_frames(fo, want_stats=False)
            g.integrate_frames(fg, want_stats=False)
        sched.call(ps)
        i += k
        last = stamps[i - 1]
        r = rng.random()
        if r < 0.25:
            o.update_tracking(last)
            g.update_tracking(last)
        elif r < 0.35:
            o.update_tracking(last)
            g.update_tracking(last)
            ro, rg = o.reset_inactive(), g.reset_inactive()
            np.testing.assert_array_equal(ro[np.lexsort(ro.T)], rg[np.lexsort(rg.T)])
            o.clear_updated()
            g.clear_updated()
        elif r < 0.45 and i < n:
            dh, lh = d[i].cpu().numpy(), l[i].cpu().numpy()
            io, _, _ = o.detect_motion(o.make_frame(dh, poses[i], stamps[i], label=lh))
            ig, _, _ = g.detect_motion(g.make_frame(dh, poses[i], stamps[i], label=lh))
            np.testing.assert_array_equal(io, ig)
            o.integrate_frame(o.make_frame(dh, poses[i], stamps[i], label=lh, mask=capi.MASK_LAST_DETECTION), want_stats=False)
            g.integrate_frames([g.make_frame(d[i].data_ptr(), poses[i], stamps[i], label=l[i].data_ptr(), mask=capi.MASK_LAST_DETECTION,
                                             memory=capi.MEM_DEVICE)], want_stats=False)
            sched.call([poses[i]])
            i += 1
        if checkpoints and rng.random() < 0.3:
            g.synchronize()
            keep.clear()
            hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"fuzz {seed} at frame {i}")
    g.synchronize()
    assert jumped and any(len(c) > (sum(x[0] for x in c) + 31) // 32 for c in sched.calls), "no split batch"
    sched.assert_covers()
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"fuzz {seed} end")
    assert o.map_checksum() == g.map_checksum()


def test_long_extractor_call_without_allocation_equals_oracle(oracle_lib, product_lib):
    """The extractor's map (vps 8, binary semantics, no tracking, pre-allocated box): one 100-frame call with
    allocate_blocks = False, device frames, no stats."""
    cam, poses, stamps, d, l = fuzz_stream()
    mc = capi.default_map_config(voxel_size=0.04, vps=8, trunc=0.08, with_tracking=False, max_blocks=45000)
    ic = capi.default_integrator_config(semantic_mode=capi.SEM_BINARY, num_threads=-1)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc, integ_cfg=ic)
    g = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=mc, integ_cfg=ic)
    bs = 0.04 * 8
    lo, hi = np.floor(np.array([2.0, 2.0, -0.3]) / bs).astype(int), np.floor(np.array([14.0, 10.0, 3.0]) / bs).astype(int)
    for h in (o, g):
        h.allocate_box(lo, hi)
    sched = Schedule(cam, bs)
    n, tid = 100, 9
    for b0 in range(0, n, K_MAX_BATCH):
        idx = range(b0, min(b0 + K_MAX_BATCH, n))
        o.integrate_frames([o.make_frame(d[i].cpu().numpy(), poses[i], stamps[i], object_image=l[i].cpu().numpy(), target_id=tid)
                            for i in idx], allocate_blocks=False, want_stats=False)
    g.integrate_frames([g.make_frame(d[i].data_ptr(), poses[i], stamps[i], object_image=l[i].data_ptr(), target_id=tid,
                                     memory=capi.MEM_DEVICE) for i in range(n)], allocate_blocks=False, want_stats=False)
    sched.call(poses[:n], allocate=False)
    g.integrate_frames([g.make_frame(d[n].data_ptr(), poses[n], stamps[n], object_image=l[n].data_ptr(), target_id=tid,
                                     memory=capi.MEM_DEVICE)], allocate_blocks=False, want_stats=False)
    o.integrate_frame(o.make_frame(d[n].cpu().numpy(), poses[n], stamps[n], object_image=l[n].cpu().numpy(), target_id=tid),
                      allocate_blocks=False, want_stats=False)
    sched.call(poses[n:n + 1], allocate=False)
    g.synchronize()
    sched.assert_covers()
    bo = o.export_blocks()
    assert (bo.semantic_label == 1).sum() > 1000
    hs.assert_blocks_equal(bo, g.export_blocks(), exact_float=True, what="extractor 100-frame call")
