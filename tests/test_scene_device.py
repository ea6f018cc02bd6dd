"""Prepared scenes from device memory (include/ray_b200.h ray_b200_prepare_scene_device, ray_b200_prepared_update,
ray_b200_prepared_spheres): a prepared scene built or rebuilt from sphere records in a CUDA buffer is, bit for bit, the
one prepare_scene makes from the same records on the host, with no record copied host -> device.

On the CPU: the Python argument checks, and the premises of the GPU tests (the animation's records are in range, and
each step's oracle frame differs from the frame of the records before it, so a stale tree cannot pass).  On the GPU,
every comparison is bit for bit (NaN-aware for float frames): against the host-array route and the CPU oracle, on every
consumer of a prepared scene, through an animation of updates, around frames in flight, the learned claim order,
store / restore, reupload, host_build contexts, the records read back, and every error."""
import ctypes as C

import numpy as np
import pytest

import limit_scenes as LS
from oracle import pyoracle as O
from ray_query_cases import _dev, _np, _torch, bits_differ, random_rays
from test_input_ranges import ALL_SCENES, _builtin, assert_frame, frame_size

MAX_N = 1 << 26

# ------------------------------------------------------------------------------------------ scenes


def _finite(name):
    s, c = ALL_SCENES[name]()
    return bool(np.isfinite(s).all())


SCENES = ["rgbbox", "irreg"] + [n for n in ALL_SCENES if _finite(n)] + ["comb_deepest", "random_2^20"]


def scene_case(name):
    """(spheres [n, 7], cam7, h, w) of a scene of SCENES"""
    if name in ("rgbbox", "irreg"):
        s, c = _builtin(name)
        return s, c, 37, 53
    if name == "comb_deepest":
        s, _ = LS.comb_scene(1 << 18)      # cluster leaves at depth 48, the deepest tree test_limits.py builds
        return s, LS.COMB_CAM, 48, 64
    if name == "random_2^20":
        s, c = O.Scene.random(1 << 20, seed=7).arrays()
        return s, c, 48, 64
    s, c = ALL_SCENES[name]()
    return (s, c) + frame_size(name)


ANIM_H, ANIM_W = 48, 64


def animation():
    """[(spheres, cam7 or None)]: the records of prepare_scene_device, then those of 9 updates (None keeps the camera):
    moving centres, changing colours and radii, a camera change, and n going 2 -> 2^16 -> 3 -> irreg's count."""
    rng = np.random.default_rng(2026)
    rg, rg_cam = _builtin("rgbbox")
    ir, ir_cam = _builtin("irreg")
    rnd, rnd_cam = O.Scene.random(1 << 16, seed=3).arrays()
    f = np.float32
    steps = [(rg.copy(), rg_cam.copy())]
    s = rg.copy()
    s[:, :3] += rng.uniform(-2, 2, (len(s), 3)).astype(f)                 # centres move
    steps.append((s, None))
    s = s.copy()
    s[:, 3:6] = s[::-1, 3:6] * f(0.75)                                    # colours change
    steps.append((s, None))
    s = s.copy()
    s[:, 6] *= f(0.6)                                                     # radii change
    steps.append((s, None))
    cam = rg_cam.copy()
    cam[0:3] += f([6, -3, 4])                                             # the camera moves
    cam[6] = f(50)
    s = s.copy()
    s[:, :3] += f([0.5, 0.25, -0.5])
    steps.append((s, cam))
    steps.append((np.ascontiguousarray(s[[3, 9]] + f([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])), None))   # n = 2
    big = rnd.copy()
    big[:, :3] += rng.normal(0, 4, (len(big), 3)).astype(f)                # n = 2^16
    steps.append((big, rnd_cam.copy()))
    steps.append((np.ascontiguousarray(big[np.argsort(big[:, 2])[-3:]] * f([1, 1, 1, 1, 1, 1, 40])), None))  # n = 3
    m = ir.copy()
    m[:, :3] += rng.uniform(-1, 1, (len(m), 3)).astype(f)                 # irreg's count
    steps.append((m, ir_cam.copy()))
    m = m.copy()
    m[:, 1] += f(1.5)
    steps.append((m, None))
    return steps


def cameras(steps):
    """The camera in effect after each step."""
    out, cam = [], None
    for _, c in steps:
        cam = c if c is not None else cam
        out.append(cam)
    return out


def oracle_pixels(s, c, h=ANIM_H, w=ANIM_W, spp=1):
    return O.Scene.custom(s, c).prepare(h, w).render(h, w, spp=spp)[0]


# ------------------------------------------------------------------------------------------ CPU


class NoContext:
    device = 0


class NoScene:
    ctx = NoContext()


def test_python_argument_checks(R):
    torch = _torch()
    s, c = _builtin("rgbbox")
    bad_spheres = [np.ascontiguousarray(s), None, torch.from_numpy(s.copy()), torch.from_numpy(s.astype(np.float64)),
                   torch.empty((4, 7), device="meta"), torch.from_numpy(s.copy())[:, :6]]
    for bad in bad_spheres:
        with pytest.raises(ValueError):
            R.Context.prepare_scene_device(NoContext(), 8, 8, bad, c)
        with pytest.raises(ValueError):
            R.PreparedScene.update(NoScene(), bad)
        with pytest.raises(ValueError):
            R.PreparedScene.update(NoScene(), bad, c)
    for bad_cam in (c[:6], c.astype(np.int32), np.stack([c, c]), torch.empty(7, device="meta"), None):
        with pytest.raises(ValueError):
            R.Context.prepare_scene_device_from_ptr(NoContext(), 8, 8, 0, 2, bad_cam)
    assert R._camera7(torch.from_numpy(c.astype(np.float64))).dtype == np.float32
    if not torch.cuda.is_available():
        return
    t = _dev(s)

    class OtherDevice:
        device = 1

    for bad in (t.double(), t[:, :6], t.reshape(7, -1).t(), t.reshape(-1), t.cpu(), t[::2]):
        with pytest.raises(ValueError):
            R.Context.prepare_scene_device(NoContext(), 8, 8, bad, c)
        with pytest.raises(ValueError):
            R.PreparedScene.update(NoScene(), bad)
    with pytest.raises(ValueError):
        R.Context.prepare_scene_device(OtherDevice(), 8, 8, t, c)
    with pytest.raises(ValueError):
        R.Context.prepare_scene_device(NoContext(), 8, 8, t, torch.from_numpy(c).cuda())


def test_animation_premises():
    """Every n the animation visits is in [2, 2^26]; it grows and shrinks as stated; every step's records give an oracle
    frame other than the records before it under the same camera (a stale tree renders the latter); and the camera
    change changes the frame of the same records."""
    steps = animation()
    cams = cameras(steps)
    ns = [len(s) for s, _ in steps]
    assert len(steps) - 1 >= 8
    assert all(2 <= n <= MAX_N for n in ns)
    assert ns[5:9] == [2, 1 << 16, 3, len(_builtin("irreg")[0])]
    assert any(c is not None for _, c in steps[1:]) and any(c is None for _, c in steps[1:])
    for k in range(1, len(steps)):
        new = oracle_pixels(steps[k][0], cams[k])
        stale = oracle_pixels(steps[k - 1][0], cams[k])
        assert (new != stale).sum() > 0, f"step {k}: the moved records render like the records before them"
    k = next(k for k in range(1, len(steps)) if steps[k][1] is not None and len(steps[k][0]) == len(steps[k - 1][0]))
    assert (oracle_pixels(steps[k][0], cams[k]) != oracle_pixels(steps[k][0], cams[k - 1])).sum() > 0
    for name in SCENES:
        s, c, h, w = scene_case(name)
        assert 2 <= len(s) <= MAX_N and np.isfinite(s).all(), name


# ------------------------------------------------------------------------------------------ GPU helpers


def frame(ctx, pr, h, w, spp=1):
    torch = _torch()
    pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
    rgb = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb)


def assert_same_scene(got, want, what):
    """info, dump and packed of two prepared scenes, bit for bit"""
    gi, wi = got.info(), want.info()
    for k in ("n_leaves", "n_inner", "max_depth", "refit_sweeps", "stale_nodes", "smem_nodes"):
        assert gi[k] == wi[k], f"{what}: info {k} {gi[k]} != {wi[k]}"
    for k in ("root_box", "camera"):
        assert bits_differ(gi[k], wi[k]) == 0, f"{what}: info {k}"
    gd, wd = got.dump(), want.dump()
    for k in gd:
        np.testing.assert_array_equal(gd[k].view(np.uint32), wd[k].view(np.uint32), err_msg=f"{what}: dump {k}")
    gp, wp = got.packed(), want.packed()
    for k in gp:
        np.testing.assert_array_equal(gp[k].view(np.uint32), wp[k].view(np.uint32), err_msg=f"{what}: packed {k}")


def assert_same_frames(ctx, got, want, h, w, spps=(1, 16), what=""):
    for spp in spps:
        gp, gr = frame(ctx, got, h, w, spp)
        wp, wr = frame(ctx, want, h, w, spp)
        assert_frame(gp, gr, wp, wr, f"{what} spp {spp}")


def host_route(ctx, h, w, s, c):
    sc = ctx.scene_from_arrays(s, c)
    pr = ctx.prepare_scene(h, w, sc)
    sc.free()
    return pr


def state(ctx, pr, h, w):
    return pr.info(), pr.dump(), pr.packed(), frame(ctx, pr, h, w, 4)


def assert_state(ctx, pr, h, w, st, what):
    info, dump, packed, (pix, rgb) = st
    now = state(ctx, pr, h, w)
    for k in ("n_leaves", "max_depth", "stale_nodes"):
        assert now[0][k] == info[k], what
    assert bits_differ(now[0]["camera"], info["camera"]) == 0, what
    for a, b in ((now[1], dump), (now[2], packed)):
        for k in a:
            np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=what)
    assert_frame(now[3][0], now[3][1], pix, rgb, what)


# ------------------------------------------------------------------------------------------ GPU: exactness


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_device_prepare_equals_host_route_and_oracle(R, name):
    s, c, h, w = scene_case(name)
    with R.Context() as ctx:
        pr = ctx.prepare_scene_device(h, w, _dev(s), c)
        want = host_route(ctx, h, w, s, c)
        assert_same_scene(pr, want, name)
        assert pr.upload_bytes() == 0 and want.upload_bytes() == 28 * len(s)
        assert pr.device_bytes() == want.device_bytes()
        o = O.Scene.custom(s, c).prepare(h, w)
        od = o.dump()
        gd = pr.dump()
        for k in ("morton", "perm", "left", "right", "parent"):
            np.testing.assert_array_equal(gd[k], od[k], err_msg=f"{name} {k} vs oracle")
        np.testing.assert_array_equal(gd["boxes"].view(np.uint32), od["boxes"].view(np.uint32))
        for spp in (1, 16):
            pix, rgb = frame(ctx, pr, h, w, spp)
            wp, wr = frame(ctx, want, h, w, spp)
            assert_frame(pix, rgb, wp, wr, f"{name} spp {spp} vs host route")
            op, orgb, _ = o.render(h, w, spp=spp, want_rgb=True)
            assert_frame(pix, rgb, op, orgb, f"{name} spp {spp} vs oracle")


@pytest.mark.gpu
def test_every_consumer_on_a_device_born_scene(R):
    """Ray queries (per call and ranged), render_views, render_gbuffer, render_accumulate and an adaptive chain on a
    device-born scene equal the same calls on the host-built equivalent."""
    torch = _torch()
    s, c = _builtin("irreg")
    s = s.copy()
    s[:, :3] += np.float32([0.25, -0.5, 0.125])
    h, w = 96, 128
    with R.Context() as ctx:
        pd = ctx.prepare_scene_device(h, w, _dev(s), c)
        ph = host_route(ctx, h, w, s, c)
        rays = _dev(random_rays(s, 8192, 5))
        lo = np.random.default_rng(6).uniform(0, 2, 8192).astype(np.float32)
        r8 = np.concatenate([_np(rays)[:, :3], lo[:, None], _np(rays)[:, 3:], (lo + 40)[:, None]], 1)
        rays8 = _dev(r8)

        def results(pr):
            out = {}
            for tag, rr in (("call", rays), ("ranged", rays8)):
                hits = ctx.trace_hits(pr, rr)
                out.update({f"hits_{tag}_{k}": _np(v) for k, v in hits.items()})
                out[f"occ_{tag}"] = _np(ctx.trace_occluded(pr, rr))
                multi = ctx.trace_multi_hits(pr, rr, 4)
                out.update({f"multi_{tag}_{k}": _np(v) for k, v in multi.items()})
            rgb, seg = ctx.trace_paths(pr, rays)
            out["paths_rgb"], out["paths_seg"] = _np(rgb), _np(seg)
            moved = c.copy()
            moved[0:3] += np.float32([3, 2, -1])
            vp, vr = ctx.render_views(pr, np.stack([c, moved]), h, w, spp=3, want_rgb=True)
            out["views_pix"], out["views_rgb"] = _np(vp), _np(vr)
            out.update({f"gbuffer_{k}": _np(v) for k, v in ctx.render_gbuffer(pr, h, w, 3).items()})
            accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
            for a, b in ((0, 1), (1, 5)):
                pix, rgb = ctx.render_accumulate(pr, accum, a, b, want_rgb=True)
            out["accum_pix"], out["accum_rgb"] = _np(pix), _np(rgb)
            acc = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")   # pixels never selected keep these
            m2 = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
            counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
            pix = torch.zeros((h, w), dtype=torch.int32, device="cuda")
            gen = torch.Generator(device="cuda").manual_seed(4)
            for n_add in (2, 1, 3):
                mask = torch.rand((h, w), device="cuda", generator=gen) < 0.5
                ctx.render_adaptive(pr, acc, counts, n_add, mask=mask, pixels=pix, m2=m2)
            sel, n_sel = ctx.adaptive_select(acc, m2, counts, 0.05, 0.1, 2, 8)
            out.update(adaptive_acc=_np(acc), adaptive_m2=_np(m2), adaptive_counts=_np(counts), adaptive_pix=_np(pix),
                       adaptive_sel=_np(sel), adaptive_n=_np(n_sel))
            return out

        got, want = results(pd), results(ph)
        for k in want:
            g, v = got[k], want[k]
            if v.dtype == np.float32:
                assert bits_differ(g, v) == 0, k
            else:
                np.testing.assert_array_equal(g, v, err_msg=k)
        assert (want["hits_call_sphere"] >= 0).sum() > 100 and want["occ_ranged"].any()


# ------------------------------------------------------------------------------------------ GPU: animation


@pytest.mark.gpu
def test_animation_updates_equal_fresh_prepares(R):
    steps = animation()
    cams = cameras(steps)
    h, w = ANIM_H, ANIM_W
    with R.Context() as ctx:
        pr = ctx.prepare_scene_device(h, w, _dev(steps[0][0]), steps[0][1])
        for k, (s, c) in enumerate(steps):
            if k > 0:
                pr.update(_dev(s), c)
            want = host_route(ctx, h, w, s, cams[k])
            assert_same_scene(pr, want, f"step {k}")
            assert_same_frames(ctx, pr, want, h, w, what=f"step {k}")
            pix, rgb = frame(ctx, pr, h, w, 1)
            op, orgb, _ = O.Scene.custom(s, cams[k]).prepare(h, w).render(h, w, want_rgb=True)
            assert_frame(pix, rgb, op, orgb, f"step {k} vs oracle")
            assert pr.upload_bytes() == 0, f"step {k}"
            got_s, got_c = pr.spheres()
            np.testing.assert_array_equal(_np(got_s).view(np.uint32), s.view(np.uint32), err_msg=f"step {k} spheres")
            np.testing.assert_array_equal(got_c.view(np.uint32), cams[k].view(np.uint32), err_msg=f"step {k} camera")
            want.free()


# ------------------------------------------------------------------------------------------ GPU: ordering


@pytest.mark.gpu
def test_a_tensor_written_on_torchs_stream_just_before_update_is_built(R):
    torch = _torch()
    s0, c = _builtin("irreg")
    s1 = s0.copy()
    s1[:, :3] *= np.float32(0.75)
    h, w = 64, 96
    with R.Context() as ctx:
        pr = ctx.prepare_scene_device(h, w, _dev(s0), c)
        src = _dev(s1)
        buf = _dev(s0)
        torch.cuda.synchronize()
        torch.cuda._sleep(100_000_000)    # keeps torch's stream busy, so the copy below lands well after the call is made
        buf.copy_(src)
        pr.update(buf)
        want = host_route(ctx, h, w, s1, c)
        assert_same_scene(pr, want, "update after a torch write")
        assert_same_frames(ctx, pr, want, h, w, (1,))
        # the same for prepare_scene_device
        torch.cuda._sleep(100_000_000)
        buf.copy_(_dev(s0))
        pd = ctx.prepare_scene_device(h, w, buf, c)
        assert_same_scene(pd, host_route(ctx, h, w, s0, c), "prepare after a torch write")


@pytest.mark.gpu
def test_frames_enqueued_before_an_update_render_the_old_records(R):
    torch = _torch()
    s0, c = _builtin("irreg")
    s1 = s0.copy()
    s1[:, :3] += np.float32([2, 1, -1])
    h, w, spp = 500, 500, 4
    with R.Context() as ctx:
        old, new = host_route(ctx, h, w, s0, c), host_route(ctx, h, w, s1, c)
        want_old, want_new = frame(ctx, old, h, w, spp)[0], frame(ctx, new, h, w, spp)[0]
        assert (want_old != want_new).any()
        outs = [torch.empty((h, w), dtype=torch.int32, device="cuda") for _ in range(6)]
        torch.cuda.synchronize()
        # one lane: render_into, then update at once
        pr = ctx.prepare_scene_device(h, w, _dev(s0), c)
        ctx.render_into(outs[0].data_ptr(), h, w, pr, spp=spp)
        pr.update(_dev(s1))
        ctx.render_into(outs[1].data_ptr(), h, w, pr, spp=spp)
        ctx.sync()
        assert (_np(outs[0]) == want_old).all() and (_np(outs[1]) == want_new).all()
        # batches with pipelined submission, frames on both lanes, an update between them
        for pipelined in (False, True):
            pr.update(_dev(s0))
            ctx.set_pipeline(pipelined)
            job = lambda o: dict(prepared=pr, h=h, w=w, out_dev=o.data_ptr(), spp=spp)
            ctx.render_batch([job(outs[2]), job(outs[3])])
            pr.update(_dev(s1))
            ctx.render_batch([job(outs[4]), job(outs[5])])
            if pipelined:
                ctx.pipeline_join()
            ctx.sync()
            ctx.set_pipeline(False)
            for k, want in ((2, want_old), (3, want_old), (4, want_new), (5, want_new)):
                assert (_np(outs[k]) == want).all(), f"pipelined={pipelined} frame {k}"


@pytest.mark.gpu
def test_freeing_the_records_after_the_call_changes_nothing(R):
    torch = _torch()
    s0, c = _builtin("rgbbox")
    s1 = s0.copy()
    s1[:, 6] *= np.float32(1.25)
    h, w = 64, 96
    with R.Context() as ctx:
        t = _dev(s0)
        pr = ctx.prepare_scene_device_from_ptr(h, w, t.data_ptr(), len(s0), c)
        del t
        junk = torch.full((len(s0), 7), float("nan"), device="cuda")
        assert_same_frames(ctx, pr, host_route(ctx, h, w, s0, c), h, w, (1,), "after freeing the prepare's records")
        t = _dev(s1)
        pr.update_from_ptr(t.data_ptr(), len(s1))
        del t
        junk2 = torch.full((len(s1), 7), float("nan"), device="cuda")
        want = host_route(ctx, h, w, s1, c)
        assert_same_scene(pr, want, "after freeing the update's records")
        assert_same_frames(ctx, pr, want, h, w, (1, 16))
        del junk, junk2


# ------------------------------------------------------------------------------------------ GPU: context state


@pytest.mark.gpu
def test_learned_order_and_context_state(R):
    """The first two frames after an update plan and launch as a freshly prepared scene's first two frames; the update
    leaves last_plan and last_render_ms unchanged and counts the build's launches as prepare_scene_device does;
    spheres() counts one launch."""
    torch = _torch()
    s0, c = _builtin("irreg")
    s1 = s0.copy()
    s1[:, :3] += np.float32([1, 0.5, 0])
    h, w, spp = 300, 400, 2
    out = torch.empty((h, w), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def frames(ctx, pr, k):
        got = []
        for _ in range(k):
            n0 = ctx.launch_count()
            ctx.render_into(out.data_ptr(), h, w, pr, spp=spp)
            ctx.sync()
            got.append((ctx.launch_count() - n0, ctx.last_plan(), _np(out).copy()))
        return got

    with R.Context(learn_order=1) as ctx:
        pr = ctx.prepare_scene_device(h, w, _dev(s0), c)
        frames(ctx, pr, 3)                     # records, then uses, the old records' claim order
        fresh = host_route(ctx, h, w, s1, c)
        want = frames(ctx, fresh, 2)
        fresh.free()
        plan, ms = ctx.last_plan(), ctx.last_render_ms()
        d = _dev(s1)
        n0 = ctx.launch_count()
        pr.update(d)
        n_update = ctx.launch_count() - n0
        assert ctx.last_plan() == plan and ctx.last_render_ms() == ms
        n0 = ctx.launch_count()
        other = ctx.prepare_scene_device(h, w, d, c)
        assert n_update == ctx.launch_count() - n0 > 0
        assert ctx.last_plan() == plan and ctx.last_render_ms() == ms
        n0 = ctx.launch_count()
        other.spheres()
        assert ctx.launch_count() - n0 == 1
        other.free()
        got = frames(ctx, pr, 2)
    for k in range(2):
        assert got[k][0] == want[k][0], f"frame {k}: {got[k][0]} launches, a fresh scene's frame {k} has {want[k][0]}"
        assert got[k][1] == want[k][1], f"frame {k}: plan"
        assert (got[k][2] == want[k][2]).all()


# ------------------------------------------------------------------------------------------ GPU: other paths


@pytest.mark.gpu
def test_store_restore_reupload_and_host_build(R):
    s0, c0 = _builtin("rgbbox")
    s1, c1 = _builtin("irreg")
    s1 = s1.copy()
    s1[:, :3] -= np.float32(0.5)
    h, w = 48, 80
    with R.Context() as ctx, R.Context(host_build=1) as ctx_h:
        want = host_route(ctx, h, w, s1, c1)
        # a scene prepared from host arrays, then updated: its stale host copy must not be stored or re-uploaded
        for born in ("host", "device"):
            pr = host_route(ctx, h, w, s0, c0) if born == "host" else ctx.prepare_scene_device(h, w, _dev(s0), c0)
            pr.update(_dev(s1), c1)
            restored = ctx.restore_prepared_scene(pr.store())
            assert_same_scene(restored, want, f"{born}: restored")
            assert_same_frames(ctx, restored, want, h, w, what=f"{born}: restored")
            pr.reupload()
            assert pr.upload_bytes() == 0
            assert_same_scene(pr, want, f"{born}: re-uploaded")
            assert_same_frames(ctx, pr, want, h, w, what=f"{born}: re-uploaded")
        # host_build: the records are read back and the host builder runs; the same scene
        ph = ctx_h.prepare_scene_device(h, w, _dev(s0), c0)
        assert_same_scene(ph, host_route(ctx, h, w, s0, c0), "host_build prepare")
        ph.update(_dev(s1), c1)
        assert_same_scene(ph, want, "host_build update")
        assert ph.upload_bytes() == ph.device_bytes() > 0
        pix, rgb = frame(ctx_h, ph, h, w, 16)
        wp, wr = frame(ctx, want, h, w, 16)
        assert_frame(pix, rgb, wp, wr, "host_build frame")
        assert_same_scene(ctx_h.restore_prepared_scene(ph.store()), want, "host_build restored")
        ph.reupload()
        assert_same_scene(ph, want, "host_build re-uploaded")
        got_s, got_c = ph.spheres()
        np.testing.assert_array_equal(_np(got_s).view(np.uint32), s1.view(np.uint32))


@pytest.mark.gpu
def test_spheres_round_trip_exactly(R):
    """spheres() gives back every bit of the records last given: signed zeros, subnormals and NaN payloads in the
    colours included, for device-born, updated and host-prepared scenes."""
    s, c = _builtin("irreg")
    s = s.copy()
    s[0, 0] = np.float32(-0.0)
    s[1, 3:6] = np.uint32([0x7FC00001, 0xFFA5A5A5, 0x00000001]).view(np.float32)
    s[2, 6] = np.float32(-0.0)
    h, w = 32, 48
    with R.Context() as ctx:
        for pr in (ctx.prepare_scene_device(h, w, _dev(s), c), host_route(ctx, h, w, s, c)):
            got_s, got_c = pr.spheres()
            np.testing.assert_array_equal(_np(got_s).view(np.uint32), s.view(np.uint32))
            np.testing.assert_array_equal(got_c.view(np.uint32), c.view(np.uint32))
            two = s[[5, 1]].copy()
            pr.update(_dev(two))
            got_s, got_c = pr.spheres()
            np.testing.assert_array_equal(_np(got_s).view(np.uint32), two.view(np.uint32))
            np.testing.assert_array_equal(got_c.view(np.uint32), c.view(np.uint32))


# ------------------------------------------------------------------------------------------ GPU: errors


@pytest.mark.gpu
def test_errors_leave_the_scene_unchanged_and_usable(R):
    torch = _torch()
    s0, c = _builtin("irreg")
    s1 = s0.copy()
    s1[:, :3] += np.float32(1)
    h, w = 40, 56
    host = np.ascontiguousarray(s1)
    with R.Context() as ctx:
        L = ctx.lib
        pr = ctx.prepare_scene_device(h, w, _dev(s0), c)
        before = state(ctx, pr, h, w)
        d = _dev(s1)
        cam = np.ascontiguousarray(c)
        out = C.c_void_p(None)
        calls = {
            "update n = 1": lambda: L.ray_b200_prepared_update(ctx.handle, pr.handle, d.data_ptr(), 1, None),
            "update n = 0": lambda: L.ray_b200_prepared_update(ctx.handle, pr.handle, d.data_ptr(), 0, None),
            "update n = 2^26 + 1": lambda: L.ray_b200_prepared_update(ctx.handle, pr.handle, d.data_ptr(), MAX_N + 1, None),
            "update NULL spheres": lambda: L.ray_b200_prepared_update(ctx.handle, pr.handle, None, len(s1), None),
            "update NULL scene": lambda: L.ray_b200_prepared_update(ctx.handle, None, d.data_ptr(), len(s1), None),
            "update host memory": lambda: L.ray_b200_prepared_update(ctx.handle, pr.handle, host.ctypes.data, len(s1), None),
            "prepare NULL out0": lambda: L.ray_b200_prepare_scene_device(ctx.handle, None, h, w, d.data_ptr(), len(s1), cam.ctypes.data),
            "prepare NULL cam7": lambda: L.ray_b200_prepare_scene_device(ctx.handle, C.byref(out), h, w, d.data_ptr(), len(s1), None),
            "prepare NULL spheres": lambda: L.ray_b200_prepare_scene_device(ctx.handle, C.byref(out), h, w, None, len(s1), cam.ctypes.data),
            "prepare h = 0": lambda: L.ray_b200_prepare_scene_device(ctx.handle, C.byref(out), 0, w, d.data_ptr(), len(s1), cam.ctypes.data),
            "prepare w < 0": lambda: L.ray_b200_prepare_scene_device(ctx.handle, C.byref(out), h, -1, d.data_ptr(), len(s1), cam.ctypes.data),
            "prepare n = 1": lambda: L.ray_b200_prepare_scene_device(ctx.handle, C.byref(out), h, w, d.data_ptr(), 1, cam.ctypes.data),
            "prepare n = 2^26 + 1": lambda: L.ray_b200_prepare_scene_device(ctx.handle, C.byref(out), h, w, d.data_ptr(), MAX_N + 1, cam.ctypes.data),
            "prepare host memory": lambda: L.ray_b200_prepare_scene_device(ctx.handle, C.byref(out), h, w, host.ctypes.data, len(s1), cam.ctypes.data),
            "spheres NULL scene": lambda: L.ray_b200_prepared_spheres(ctx.handle, None, d.data_ptr(), cam.ctypes.data),
        }
        for what, call in calls.items():
            assert call() != 0, what
            msg = ctx.get_error()
            assert msg, what
            if "n = " in what:
                assert "spheres" in msg, (what, msg)
            assert out.value is None, what
            assert_state(ctx, pr, h, w, before, what)
        np.testing.assert_array_equal(_np(d).view(np.uint32), s1.view(np.uint32))
        pr.update(d)          # and still usable
        assert_same_scene(pr, host_route(ctx, h, w, s1, c), "after the errors")
        with pytest.raises(R.RayError, match="spheres"):
            pr.update(d[:1])
        assert_same_scene(pr, host_route(ctx, h, w, s1, c), "after a Python-level error")


@pytest.mark.gpu
def test_multi_gpu_contexts_are_rejected(R):
    torch = _torch()
    if torch.cuda.device_count() < 2:
        pytest.skip("a RAY_GPUS > 1 context needs two GPUs")
    s0, c = _builtin("rgbbox")
    h, w = 32, 48
    with R.Context(gpus=2) as ctx:
        with pytest.raises(R.RayError, match="RAY_GPUS"):
            ctx.prepare_scene_device(h, w, _dev(s0), c)
        pr = host_route(ctx, h, w, s0, c)
        before = pr.dump(), pr.packed()
        with pytest.raises(R.RayError, match="RAY_GPUS"):
            pr.update(_dev(s0[:5]))
        for a, b in zip((pr.dump(), pr.packed()), before):
            for k in a:
                np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32))
        img = ctx.render(h, w, pr)
        ctx.sync()
        assert (img.values() == O.Scene.custom(s0, c).prepare(h, w).render(h, w)[0]).all()
