"""Scene batches (include/ray_b200.h "scene batches"): B scenes of n spheres each, built in one pass from one CUDA tensor
and rendered in one launch.  Member b is bit for bit the prepared scene prepare_scene_device makes of scene b's records,
and frame b of a batch render is render_into of member b, bit for bit (NaN-aware for float frames).

On the CPU: the Python argument checks and the camera table.  On the GPU: the build against the single-scene route, the
host builder and the oracle, on mixed batches; frames against members, independently prepared scenes and the oracle, on
every plan the kind reaches; updates, ordering, memory and errors."""
import numpy as np
import pytest

import limit_scenes as LS
from oracle import pyoracle as O
from ray_query_cases import _dev, _np, _torch, bits_differ
from test_input_ranges import ALL_SCENES, _builtin, assert_frame

SENTINEL = 0x7FA5A5A5
STAGING = {(0, 0): "partial", (1, 0): "nodes", (1, 1): "whole"}


# ------------------------------------------------------------------------------------------ batches


def random_batch(B, n, seed=1):
    """B scenes of n random spheres each (different extents, so boxes and Morton keys differ per scene), and cameras."""
    rng = np.random.default_rng(seed)
    side = (2.2 * n ** (1 / 3)) * rng.uniform(0.5, 2.0, B).astype(np.float32)
    s = np.empty((B, n, 7), np.float32)
    s[:, :, 0:3] = rng.uniform(-0.5, 0.5, (B, n, 3)).astype(np.float32) * side[:, None, None]
    s[:, :, 3:6] = rng.uniform(0.2, 0.95, (B, n, 3))
    s[:, :, 6] = rng.uniform(0.4, 1.2, (B, n)) * (side[:, None] / side.mean())
    cams = np.zeros((B, 7), np.float32)
    cams[:, 0] = 0.35 * side
    cams[:, 1] = 0.45 * side
    cams[:, 2] = 1.7 * side
    cams[:, 6] = rng.uniform(40, 70, B)
    return s, cams


def fit(s, n):
    """s truncated or padded with far-away, tiny spheres to n records"""
    if len(s) >= n:
        return np.ascontiguousarray(s[:n])
    pad = np.zeros((n - len(s), 7), np.float32)
    pad[:, 0] = 1e4 + np.arange(n - len(s), dtype=np.float32)
    pad[:, 1] = -1e4
    pad[:, 3:6] = 0.5
    pad[:, 6] = 0.01
    return np.ascontiguousarray(np.concatenate([s, pad]), np.float32)


def mixed_batch(n):
    """Members that differ in everything that matters, side by side, each n spheres: rgbbox (stale boxes), irreg, every
    input-range scene (NaN / inf / out-of-range records), all centres coincident (flat axes), duplicates, a deep comb next
    to a shallow random scene."""
    members = []
    for name in ("rgbbox", "irreg"):
        s, c = _builtin(name)
        members.append((fit(s, n), c))
    for name in sorted(ALL_SCENES):
        s, c = ALL_SCENES[name]()
        members.append((fit(s, n), c))
    s, c = _builtin("rgbbox")
    same = np.repeat(fit(s, 1)[:1], n, 0)
    same[:, 3:6] = np.linspace(0.1, 0.9, n, dtype=np.float32)[:, None]
    members.append((same, c))                                  # all centres coincident
    dup = fit(s, max(1, n // 2))
    members.append((np.ascontiguousarray(np.concatenate([dup, dup])[:n] if 2 * len(dup) >= n else fit(dup, n)), c))
    comb, _ = LS.comb_scene(max(n, 2))
    members.append((fit(comb, n), LS.COMB_CAM))                 # deep
    r, rc = random_batch(1, n, seed=5)
    members.append((r[0], rc[0]))                               # shallow
    s = np.ascontiguousarray(np.stack([m[0] for m in members]), np.float32)
    cams = np.ascontiguousarray(np.stack([m[1] for m in members]), np.float32)
    return s, cams


# ------------------------------------------------------------------------------------------ CPU


class NoContext:
    device = 0


def test_python_argument_checks(R):
    torch = _torch()
    s, cams = random_batch(3, 5)
    bad = [s, None, torch.from_numpy(s), torch.from_numpy(s.astype(np.float64)), torch.from_numpy(s[0]),
           torch.empty((3, 5, 7), device="meta"), torch.from_numpy(s)[:, :, :6], torch.from_numpy(s[:, :1].copy())]
    for b in bad:
        with pytest.raises(ValueError):
            R.Context.prepare_scene_batch(NoContext(), 8, 8, b, cams)
    for bad_cam in (cams[:2], cams[:, :6], cams.astype(np.int32), cams[0], None):
        with pytest.raises(ValueError):
            R.scene_batch_cameras(bad_cam, 3)
    assert R.scene_batch_cameras(torch.from_numpy(cams.astype(np.float64)), 3).dtype == np.float32
    assert R.scene_batch_frames_ok(1, 1, 1) and R.scene_batch_frames_ok(1 << 25, 4, 8)
    assert not R.scene_batch_frames_ok((1 << 25) + 1, 4, 8) and not R.scene_batch_frames_ok(5, 1 << 15, 1 << 13)
    assert R.scene_batch_frames_ok(1, 1 << 15, 1 << 13) and not R.scene_batch_frames_ok(1, 0, 8)
    if not torch.cuda.is_available():
        return
    t = _dev(s)
    for b in (t.double(), t[:, :, :6], t.transpose(0, 1), t.cpu(), t[::2], t[:, :1]):
        with pytest.raises(ValueError):
            R.Context.prepare_scene_batch(NoContext(), 8, 8, b, cams)
    big = torch.empty((1 << 20, 65, 7), dtype=torch.float32, device="cuda")   # 2^26 + 2^20 spheres
    with pytest.raises(ValueError):
        R.scene_batch_rows(0, big)
    with pytest.raises(ValueError):   # 2^20 frames of 64 x 32 tiles pass 2^25 tiles
        R.Context.prepare_scene_batch(NoContext(), 256, 256, torch.empty((1 << 20, 2, 7), device="cuda"), np.zeros((1 << 20, 7)))


def test_query_name(R):
    assert R.QUERIES[9] == "scene_batch"


# ------------------------------------------------------------------------------------------ GPU helpers


def frames_of(ctx, batch, h, w, spp):
    torch = _torch()
    B = batch.shape[0]
    pix = torch.full((B, h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((B, h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    torch.cuda.synchronize()
    ctx.render_scene_batch_into(batch, h, w, spp, pix.data_ptr(), rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb), ctx.last_plan()


def frame(ctx, pr, h, w, spp):
    torch = _torch()
    pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    torch.cuda.synchronize()
    ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb)


def assert_same_scene(got, want, what):
    gi, wi = got.info(), want.info()
    for k in ("n_leaves", "n_inner", "max_depth", "refit_sweeps", "stale_nodes", "smem_nodes"):
        assert gi[k] == wi[k], f"{what}: info {k} {gi[k]} != {wi[k]}"
    for k in ("root_box", "camera"):
        assert bits_differ(gi[k], wi[k]) == 0, f"{what}: info {k}"
    for a, b, tag in ((got.dump(), want.dump(), "dump"), (got.packed(), want.packed(), "packed")):
        for k in a:
            np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=f"{what}: {tag} {k}")
    gs, gc = got.spheres()
    ws, wc = want.spheres()
    assert bits_differ(_np(gs), _np(ws)) == 0 and bits_differ(gc, wc) == 0, f"{what}: spheres"


# ------------------------------------------------------------------------------------------ GPU: build exactness


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 7, 64, 1024])
@pytest.mark.parametrize("n", [2, 3, 64, 1000])
def test_members_equal_single_scene_builds(R, B, n):
    h, w = 24, 40
    s, cams = random_batch(B, n, seed=B * 7 + n)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
        assert batch.shape == (B, n)
        check = range(B) if B <= 8 else sorted({0, 1, B // 3, B // 2, B - 2, B - 1})
        for b in check:
            m = batch.member(b)
            want = ctx.prepare_scene_device(h, w, _dev(s[b]), cams[b])
            assert_same_scene(m, want, f"B={B} n={n} member {b}")
            assert m.upload_bytes() == 0
            if n <= 64 and b < 2:
                hl = R.host_lbvh(s[b])
                d = m.dump()
                for k in ("morton", "perm", "left", "right", "parent"):
                    np.testing.assert_array_equal(d[k], hl[k], err_msg=f"{k} vs host_lbvh")
                od = O.Scene.custom(s[b], cams[b]).prepare(h, w).dump()
                np.testing.assert_array_equal(d["boxes"].view(np.uint32), od["boxes"].view(np.uint32))
            m.free(); want.free()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3, 64, 1000])
def test_mixed_batch_members(R, n):
    h, w = 48, 64
    s, cams = mixed_batch(n)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
        depths = set()
        for b in range(len(s)):
            m = batch.member(b)
            want = ctx.prepare_scene_device(h, w, _dev(s[b]), cams[b])
            assert_same_scene(m, want, f"n={n} member {b}")
            depths.add(m.info()["max_depth"])
            m.free(); want.free()
        pix, rgb, plan = frames_of(ctx, batch, h, w, 4)
        assert plan["query"] == "scene_batch"
        for b in range(len(s)):
            want = ctx.prepare_scene_device(h, w, _dev(s[b]), cams[b])
            wp, wr = frame(ctx, want, h, w, 4)
            assert_frame(pix[b], rgb[b], wp, wr, f"n={n} frame {b}")
            want.free()
        if n >= 64:
            assert len(depths) > 2, depths


@pytest.mark.gpu
def test_largest_batch(R):
    """B n = 2^26: a sample of members against their own builds."""
    B, n = 1 << 16, 1 << 10
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(3)
    s = torch.rand((B, n, 7), device="cuda", generator=gen)
    s[:, :, 0:3] *= 40.0
    s[:, :, 6] = s[:, :, 6] * 0.8 + 0.2
    cams = np.tile(np.float32([20, 30, 120, 20, 20, 20, 50]), (B, 1))
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(16, 16, s, cams)
        for b in (0, 1, B // 2 + 3, B - 1):
            m = batch.member(b)
            want = ctx.prepare_scene_device(16, 16, s[b].contiguous(), cams[b])
            assert_same_scene(m, want, f"member {b}")
            m.free(); want.free()
        pix = ctx.render_scene_batch(batch, 4, 8)
        want = ctx.prepare_scene_device(16, 16, s[B - 1].contiguous(), cams[B - 1])
        assert (_np(pix[B - 1]) == frame(ctx, want, 4, 8, 1)[0]).all()


# ------------------------------------------------------------------------------------------ GPU: render exactness


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,B,n", [(1, 1, 5, 64), (7, 13, 6, 100), (84, 84, 16, 64), (256, 256, 3, 1000), (1000, 1000, 2, 300)])
@pytest.mark.parametrize("spp", [1, 4, 16, 64])
def test_frames_equal_member_and_independent_renders(R, h, w, B, n, spp):
    if h * w * spp > 1000 * 1000 * 16:
        pytest.skip("covered at fewer samples")
    s, cams = random_batch(B, n, seed=h + spp)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
        pix, rgb, plan = frames_of(ctx, batch, h, w, spp)
        assert plan["query"] == "scene_batch"
        for b in range(B):
            m = batch.member(b)
            ind = ctx.prepare_scene_device(h, w, _dev(s[b]), cams[b])
            mp, mr = frame(ctx, m, h, w, spp)
            ip, ir = frame(ctx, ind, h, w, spp)
            assert_frame(pix[b], rgb[b], mp, mr, f"frame {b} vs member")
            assert_frame(pix[b], rgb[b], ip, ir, f"frame {b} vs independent")
            if h * w <= 100 and spp <= 16:
                op, orgb, _ = O.Scene.custom(s[b], cams[b]).prepare(h, w).render(h, w, spp, want_rgb=True)
                assert_frame(pix[b], rgb[b], op, orgb, f"frame {b} vs oracle")
            m.free(); ind.free()


def _staging(plan):
    return STAGING[(plan["all_nodes"], plan["spheres"])]


@pytest.mark.gpu
def test_every_plan_of_the_kind(R):
    """Forced staging points (partial, nodes, whole), K = 1 / 2, spread and pixel-bound, packet on and off: every variant
    the planner reaches for kSceneBatch is launched, and every frame equals render_into of the members."""
    h, w, B, n = 48, 64, 8, 60   # small enough to be staged whole next to the queues of every plan below
    s, cams = random_batch(B, n, seed=11)
    n_inner, n_leaves = B * (n - 1), B * n
    caps = {"partial": 64 * (n_inner // 3), "nodes": 64 * n_inner + 128, "whole": 64 * n_inner + 16 * n_leaves + 256}
    want = {}
    with R.Context() as ref:
        for b in range(B):
            pr = ref.prepare_scene_device(h, w, _dev(s[b]), cams[b])
            want[b] = {spp: frame(ref, pr, h, w, spp) for spp in (1, 4)}
            pr.free()
    launched = set()
    for plan_kw in (dict(wq_k=1, wq_warps=32), dict(wq_k=2, wq_warps=16)):
        for stage, cap in caps.items():
            for packet in (0, 24):
                for spp, spread in ((1, 0), (4, 1), (4, 0)):
                    with R.Context(stage_cap=cap, wq_packet=packet, wq_spread=spread, wq_ncap=256, **plan_kw) as ctx:
                        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
                        pix, rgb, plan = frames_of(ctx, batch, h, w, spp)
                        what = f"{plan_kw} {stage} packet {packet} spp {spp} spread {spread}"
                        assert plan["query"] == "scene_batch" and _staging(plan) == stage, (what, plan)
                        assert plan["k"] == plan_kw["wq_k"] and bool(plan["packet"]) == bool(packet), (what, plan)
                        launched.add((plan["k"], bool(plan["spread"]), plan["packet"] > 0, stage))
                        for b in range(B):
                            assert_frame(pix[b], rgb[b], *want[b][spp], f"{what} frame {b}")
    reachable = {(k, sp, pk, st) for k in (1, 2) for sp in (False, True) for pk in (False, True) for st in STAGING.values()}
    assert launched == reachable, reachable - launched


@pytest.mark.gpu
def test_outputs_past_4_gib(R):
    """B x h x w x 3 floats pass 4 GiB: the last frame lands at its 64-bit offset."""
    torch = _torch()
    h, w = 1024, 1024
    B = 360   # 360 x 2^20 x 12 bytes = 4.2 GiB of floats
    s, cams = random_batch(B, 8, seed=9)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
        pix = torch.empty((B, h, w), dtype=torch.int32, device="cuda")
        rgb = torch.empty((B, h, w, 3), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        ctx.render_scene_batch_into(batch, h, w, 1, pix.data_ptr(), rgb.data_ptr())
        ctx.sync()
        for b in (0, B - 1):
            pr = ctx.prepare_scene_device(h, w, _dev(s[b]), cams[b])
            wp, wr = frame(ctx, pr, h, w, 1)
            assert_frame(_np(pix[b]), _np(rgb[b]), wp, wr, f"frame {b}")
            pr.free()
        del pix, rgb


# ------------------------------------------------------------------------------------------ GPU: updates and ordering


@pytest.mark.gpu
def test_animation_by_torch_ops(R):
    torch = _torch()
    h, w, B, n = 48, 64, 6, 200
    s0, cams = random_batch(B, n, seed=21)
    with R.Context() as ctx:
        t = _dev(s0)
        batch = ctx.prepare_scene_batch(h, w, t, cams)
        prs = [ctx.prepare_scene_device(h, w, t[b].contiguous(), cams[b]) for b in range(B)]
        gen = torch.Generator(device="cuda").manual_seed(1)
        for step in range(9):
            if step > 0:
                t = t.clone()
                t[:, :, 0:3] += torch.randn((B, n, 3), device="cuda", generator=gen) * 0.5
                t[:, :, 3:6] = t[:, :, 3:6].flip(1) * 0.9
                new_cams = None if step % 3 else cams + np.float32([step, 0, 0, 0, 0, 0, 0])
                if new_cams is not None:
                    cams = new_cams
                batch.update(t, new_cams)
                for b in range(B):
                    prs[b].update(t[b].contiguous(), cams[b] if new_cams is not None else None)
            fresh = ctx.prepare_scene_batch(h, w, t, cams)
            pix, rgb, _ = frames_of(ctx, batch, h, w, 4)
            fp, fr, _ = frames_of(ctx, fresh, h, w, 4)
            assert (pix == fp).all() and bits_differ(rgb, fr) == 0, f"step {step} vs a fresh batch"
            for b in range(B):
                wp, wr = frame(ctx, prs[b], h, w, 4)
                assert_frame(pix[b], rgb[b], wp, wr, f"step {step} frame {b} vs the per-scene route")
            fresh.free()


@pytest.mark.gpu
def test_update_keeps_cameras_and_bad_update_leaves_batch(R):
    torch = _torch()
    h, w, B, n = 32, 48, 4, 50
    s, cams = random_batch(B, n, seed=3)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
        before = frames_of(ctx, batch, h, w, 1)
        m0 = batch.member(0).info()["camera"]
        batch.update(_dev(s))
        assert bits_differ(batch.member(0).info()["camera"], m0) == 0
        after = frames_of(ctx, batch, h, w, 1)
        assert (before[0] == after[0]).all()
        with pytest.raises(ValueError):
            batch.update(_dev(s[:, :n - 1].copy()))
        with pytest.raises(R.RayError):
            batch.update_from_ptr(0)
        with pytest.raises(R.RayError):
            batch.update_from_ptr(torch.from_numpy(s).data_ptr())   # plain host memory
        again = frames_of(ctx, batch, h, w, 1)
        assert (again[0] == before[0]).all() and batch.shape == (B, n)


@pytest.mark.gpu
def test_frames_in_flight_read_the_old_trees_and_free_behind_them(R):
    torch = _torch()
    h, w, B, n = 256, 256, 8, 2000
    s, cams = random_batch(B, n, seed=4)
    s2 = s.copy()
    s2[:, :, 0:3] += 3.0
    with R.Context() as ctx:
        old_want = frames_of(ctx, ctx.prepare_scene_batch(h, w, _dev(s), cams), h, w, 16)[0]
        new_want = frames_of(ctx, ctx.prepare_scene_batch(h, w, _dev(s2), cams), h, w, 16)[0]
        assert (old_want != new_want).any()
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
        a = torch.empty((B, h, w), dtype=torch.int32, device="cuda")
        b2 = torch.empty((B, h, w), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.render_scene_batch_into(batch, h, w, 16, a.data_ptr())
        batch.update(_dev(s2))
        ctx.render_scene_batch_into(batch, h, w, 16, b2.data_ptr())
        batch.free()                      # with the second render possibly still running
        ctx.sync()
        assert (_np(a) == old_want).all() and (_np(b2) == new_want).all()


@pytest.mark.gpu
def test_streams_and_pipeline_lanes(R):
    torch = _torch()
    h, w, B, n = 64, 64, 4, 300
    s, cams = random_batch(B, n, seed=8)
    with R.Context() as ctx:
        want = frames_of(ctx, ctx.prepare_scene_batch(h, w, _dev(s), cams), h, w, 4)[0]
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            ctx.set_stream(st.cuda_stream)
            t = _dev(s)
            batch = ctx.prepare_scene_batch(h, w, t, cams)
            pix = torch.empty((B, h, w), dtype=torch.int32, device="cuda")
            ctx.render_scene_batch_into(batch, h, w, 4, pix.data_ptr())
            st.synchronize()
        ctx.set_stream(None)
        assert (_np(pix) == want).all()
        ctx.set_pipeline(True)
        pr = ctx.prepare_scene_device(h, w, _dev(s[0]), cams[0])
        jobs_out = torch.empty((2, h, w), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.render_batch([dict(prepared=pr, h=h, w=w, spp=4, out_dev=jobs_out[k].data_ptr()) for k in range(2)])
        ctx.render_scene_batch_into(batch, h, w, 4, pix.data_ptr())
        batch.update(_dev(s))
        batch.free()
        ctx.pipeline_join()
        ctx.sync()
        assert (_np(pix) == want).all() and (_np(jobs_out[1]) == want[0]).all()


@pytest.mark.gpu
def test_prepared_scene_renders_unchanged_around_batch_renders(R):
    """A prepared scene's frames, launches and plans are the same with batch renders in between (its learned order stays)."""
    h, w = 96, 128
    s, cams = random_batch(4, 500, seed=12)

    def run(with_batch):
        torch = _torch()
        with R.Context() as ctx:
            pr = ctx.prepare_scene_device(h, w, _dev(s[0]), cams[0])
            batch = ctx.prepare_scene_batch(h, w, _dev(s), cams) if with_batch else None
            out = []
            for k in range(4):
                pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                n0 = ctx.launch_count()
                ctx.render_into(pix.data_ptr(), h, w, pr, spp=4)
                ctx.sync()
                out.append((ctx.launch_count() - n0, ctx.last_plan(), _np(pix)))
                if batch is not None:
                    n0 = ctx.launch_count()
                    frames_of(ctx, batch, h, w, 4)
                    assert ctx.launch_count() - n0 == 1 and ctx.last_render_ms() > 0
            return out

    got, want = run(True), run(False)
    for k in range(4):
        assert got[k][0] == want[k][0] and got[k][1] == want[k][1] and (got[k][2] == want[k][2]).all(), k


# ------------------------------------------------------------------------------------------ GPU: memory contract


@pytest.mark.gpu
def test_guarded_outputs_and_untouched_inputs(R):
    torch = _torch()
    h, w, B, n = 13, 21, 3, 40
    s, cams = random_batch(B, n, seed=5)
    G = 4096
    with R.Context() as ctx:
        t = _dev(s)
        before = _np(t).copy()
        cams_before = cams.copy()
        batch = ctx.prepare_scene_batch(h, w, t, cams)
        want = frames_of(ctx, batch, h, w, 4)
        for fill in (0x00, 0xFF):
            pix = torch.full((2 * G + B * h * w,), fill * 0x01010101 - (1 << 32 if fill else 0), dtype=torch.int32, device="cuda")
            rgb = torch.full((2 * G + B * h * w * 3,), fill * 0x01010101 - (1 << 32 if fill else 0), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            ctx.render_scene_batch_into(batch, h, w, 4, pix[G:].data_ptr(), rgb[G:].data_ptr())
            ctx.sync()
            p, r = _np(pix), _np(rgb)
            guard = np.int32(fill * 0x01010101 - (1 << 32 if fill else 0))
            assert (p[:G] == guard).all() and (p[G + B * h * w:] == guard).all(), fill
            assert (r[:G] == guard).all() and (r[G + B * h * w * 3:] == guard).all(), fill
            assert (p[G:G + B * h * w].reshape(B, h, w) == want[0]).all()
            assert bits_differ(r[G:G + B * h * w * 3].view(np.float32).reshape(B, h, w, 3), want[1]) == 0
        m = batch.member(1)
        ind = ctx.prepare_scene_device(h, w, _dev(s[1]), cams[1])
        assert_same_scene(m, ind, "member after guarded renders")
        batch.update(t)
        ctx.sync()
        assert (_np(t).view(np.uint32) == before.view(np.uint32)).all() and (cams == cams_before).all()


@pytest.mark.gpu
@pytest.mark.parametrize("poison", [0x00, 0xFF, 0x7F])
def test_outputs_do_not_depend_on_pool_contents(R, poison):
    """The stream-ordered pool the build, the update and the render allocate from is filled with the pattern before each
    (the context runs on a torch stream, where the pool's freed blocks are reused first): the frames are the same."""
    from test_memory_contract import Driver
    torch = _torch()
    h, w, B, n = 48, 64, 5, 300
    s, cams = random_batch(B, n, seed=13)
    with R.Context() as ref:
        want = frames_of(ref, ref.prepare_scene_batch(h, w, _dev(s), cams), h, w, 4)
    drv = Driver(0)
    st = torch.cuda.Stream()
    with R.Context() as ctx, torch.cuda.stream(st):
        ctx.set_stream(st.cuda_stream)
        t = _dev(s)
        st.synchronize()
        drv.poison_pool(st.cuda_stream, poison)
        batch = ctx.prepare_scene_batch(h, w, t, cams)
        drv.poison_pool(st.cuda_stream, poison)
        batch.update(t)
        drv.poison_pool(st.cuda_stream, poison)
        got = frames_of(ctx, batch, h, w, 4)
        m = batch.member(2)
        drv.poison_pool(st.cuda_stream, poison)
        assert (frame(ctx, m, h, w, 4)[0] == want[0][2]).all()
        batch.free(); m.free()
        ctx.set_stream(None)
    assert (got[0] == want[0]).all() and bits_differ(got[1], want[1]) == 0


# ------------------------------------------------------------------------------------------ GPU: errors


@pytest.mark.gpu
def test_errors_leave_the_context_usable(R):
    torch = _torch()
    h, w, B, n = 16, 16, 3, 20
    s, cams = random_batch(B, n, seed=2)
    t = _dev(s)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, t, cams)
        c = np.ascontiguousarray(cams)
        for call in (lambda: ctx.prepare_scene_batch_from_ptr(h, w, t.data_ptr(), 0, n, c[:0]),        # n_scenes < 1
                     lambda: ctx.prepare_scene_batch_from_ptr(h, w, t.data_ptr(), B, 1, c),            # n < 2
                     lambda: ctx.prepare_scene_batch_from_ptr(h, w, t.data_ptr(), 1 << 20, 65, np.zeros((1 << 20, 7), np.float32)),  # B n > 2^26
                     lambda: ctx.prepare_scene_batch_from_ptr(1 << 15, 1 << 14, t.data_ptr(), B, n, c),  # B x tiles > 2^25
                     lambda: ctx.prepare_scene_batch_from_ptr(0, w, t.data_ptr(), B, n, c),
                     lambda: ctx.prepare_scene_batch_from_ptr(h, w, 0, B, n, c),
                     lambda: ctx.prepare_scene_batch_from_ptr(h, w, s.ctypes.data, B, n, c),           # host memory
                     lambda: batch.member(-1), lambda: batch.member(B),
                     lambda: ctx.render_scene_batch_into(batch, h, w, 0, t.data_ptr()),                 # spp < 1
                     lambda: ctx.render_scene_batch_into(batch, h, w, 1, 0),
                     lambda: ctx.render_scene_batch_into(batch, 1 << 15, 1 << 14, 1, t.data_ptr())):
            with pytest.raises(R.RayError):
                call()
        assert ctx.last_plan()["query"] != "scene_batch"
        want = frames_of(ctx, batch, h, w, 1)[0]
        ctx.set_shard(0, 2)
        pix = torch.empty((B, h, w), dtype=torch.int32, device="cuda")
        for call in (lambda: ctx.render_scene_batch_into(batch, h, w, 1, pix.data_ptr()),
                     lambda: ctx.prepare_scene_batch(h, w, t, cams), lambda: batch.update(t)):
            with pytest.raises(R.RayError):
                call()
        ctx.set_shard(0, 1)
        assert (frames_of(ctx, batch, h, w, 1)[0] == want).all()
    with R.Context(host_build=1) as ctx:
        with pytest.raises(R.RayError):
            ctx.prepare_scene_batch(h, w, t, cams)
        assert (ctx.render(h, w, ctx.prepare_scene_device(h, w, t[0].contiguous(), cams[0])).values() != 0).any()
