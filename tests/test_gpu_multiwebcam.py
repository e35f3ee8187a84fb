"""Webcam pool (MultiWebcamAdaptor) and its grouped input side on the GPU.

- dboa_crop_resize_normalize_groups / dboa_keypoint_transform_groups: every active row bit-identical to the one-frame calls,
  for frames of different sizes and dtypes, boxes partly and wholly outside the frame, up- and down-scaling crops; idle frames
  (NaN-filled) not read and idle rows (a sentinel) not written; the dataprocess golden through the new entry.
- One stream is WebcamAdaptor, bit for bit, at adapt_webcam.npz's options.
- G = 4 at the golden's options: stream 0 against the golden, streams 1..3 against their own WebcamAdaptor runs; the motion term
  goes live from frame `interval` on.
- Streams that sit ticks out, change slot and meet other streams' starts and pauses; reload(g); online_adaptation end to end."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from harness import SIZES, bits, cam_options, state, webcam_pool

pytestmark = pytest.mark.gpu
SENTINEL = 0x7fc0dead                  # a NaN payload no kernel writes


# ------------------------------------------------------------------ grouped input side


def scene(G, seed):
    """G frames (sizes of SIZES, uint8 and float32 mixed) with boxes inside, partly outside and wholly outside the frame, and
    scales that up-scale (box smaller than 224) and down-scale."""
    rng = np.random.default_rng(seed)
    frames, centers, scales = [], [], []
    for g in range(G):
        H, W = SIZES[(g + seed) % len(SIZES)]
        img = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
        t = torch.from_numpy(img).cuda()
        frames.append(t if g % 2 == 0 else t.float())
        kind = (g + seed) % 4
        if kind == 0:
            c, s = [W / 2 + rng.uniform(-20, 20), H / 2 + rng.uniform(-20, 20)], min(H, W) / 200 * rng.uniform(0.3, 0.9)
        elif kind == 1:
            c, s = [rng.uniform(0, 0.1) * W, rng.uniform(0.9, 1.0) * H], min(H, W) / 200 * 0.8
        elif kind == 2:
            c, s = [W + 300.0, -250.0], 1.2                                  # wholly outside: zeros
        else:
            c, s = [rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H], 0.5  # 100-pixel box: up-scales
        centers.append(c)
        scales.append(s)
    return frames, centers, scales


@pytest.mark.parametrize('G', [1, 2, 4, 8])
def test_grouped_crop_is_the_one_frame_crop(G):
    from dynaboa_b200 import dataprocess as D
    frames, centers, scales = scene(G, G)
    ref = [D.crop(f, c, s) for f, c, s in zip(frames, centers, scales)]
    Ts = {D._tables(D._box(c, s, (224, 224))[3], 224, frames[0].device)[1].shape[1] for c, s in zip(centers, scales)}
    if G >= 4:
        assert len(Ts) > 1                                                   # the Ty of the videos differ
    out = torch.full((G, 3, 224, 224), float('nan'), device='cuda')
    D.crop_groups(frames, centers, scales, out)
    for g in range(G):
        assert torch.equal(bits(out[g]), bits(ref[g])), g
    masks = [1] if G == 1 else [1 << (G - 1), ((1 << G) - 1) & ~0b10]        # one active; all but one
    for active in masks:
        idle = [g for g in range(G) if not (active >> g) & 1]
        fr = [torch.full_like(f, float('nan'), dtype=torch.float32) if g in idle else f for g, f in enumerate(frames)]
        out = torch.empty(G, 3, 224, 224, device='cuda')
        out.view(torch.int32).fill_(SENTINEL)
        D.crop_groups(fr, centers, scales, out, active)
        torch.cuda.synchronize()
        for g in range(G):
            if g in idle:
                assert bool((out[g].view(torch.int32) == SENTINEL).all()), (bin(active), g)
            else:
                assert torch.equal(bits(out[g]), bits(ref[g])), (bin(active), g)


def test_grouped_input_side_holds_the_golden(golden):
    from dynaboa_b200 import dataprocess as D
    from oracle import dataprocess_ref as R
    gd = golden('dataprocess')
    n = len(gd['scales'])
    img = torch.from_numpy(gd['img']).cuda()
    centers, scales = [list(c) for c in gd['centers']], [float(s) for s in gd['scales']]
    out = D.crop_groups([img] * n, centers, scales, torch.empty(n, 3, 224, 224, device='cuda')).cpu().numpy()
    kp = torch.from_numpy(gd['kp']).float().cuda()
    kps = D.j2d_processing_groups(kp.expand(n, 49, 3), centers, scales, torch.empty(n, 49, 3, device='cuda')).cpu().numpy()
    for i in range(n):
        ref = R.rgb_processing(gd['img'], centers[i], scales[i])
        assert np.abs(out[i] - ref).max() < 2e-5, i
        assert np.abs(out[i][:, ::4, ::4] - gd['crops_sub'][i]).max() < 2e-5, i
        assert np.array_equal(kps[i], R.j2d_processing(gd['kp'].astype(np.float32).astype(np.float64), centers[i], scales[i])), i


@pytest.mark.parametrize('G,active', [(1, None), (3, None), (8, 0b10110101), (8, 1 << 7)])
def test_grouped_keypoints_are_the_one_stream_transform(G, active):
    from dynaboa_b200 import dataprocess as D
    frames, centers, scales = scene(G, 17 + G)
    rng = np.random.default_rng(G)
    det = np.concatenate([rng.uniform(-100, 2000, size=(G, 25, 2)), (rng.uniform(0, 1, size=(G, 25, 1)) > 0.3)], 2)
    kp = torch.from_numpy(det).float().cuda()
    out = torch.empty(G, 49, 3, device='cuda')
    out.view(torch.int32).fill_(SENTINEL)
    on = (1 << G) - 1 if active is None else active
    kin = kp.clone()
    for g in range(G):
        if not (on >> g) & 1:
            kin[g] = float('nan')
    D.j2d_processing_groups(kin, centers, scales, out, active)
    torch.cuda.synchronize()
    for g in range(G):
        if not (on >> g) & 1:
            assert bool((out[g].view(torch.int32) == SENTINEL).all()), g
            continue
        assert torch.equal(bits(out[g, :25]), bits(D.j2d_processing(kp[g], centers[g], scales[g]))), g
        assert bool((out[g, 25:] == 0).all()) and not torch.signbit(out[g, 25:]).any(), g


# ------------------------------------------------------------------ the pool
def single(tmp, gd, name, **extra):
    from dynaboa_b200.webcam import WebcamAdaptor
    return WebcamAdaptor(cam_options(tmp / name, gd, **extra))


def stream_inputs(gd, vid, n):
    """Frames and (1, 49, 3) keypoint blocks of stream `vid`: the golden's for 0, other frames and detections for the others."""
    from dynaboa_b200 import synthetic
    s = synthetic.SyntheticStream(length=n, batch_size=1, rank=vid)
    rng = np.random.default_rng(100 + vid)
    out = []
    for t in range(n):
        kp = torch.zeros(1, 49, 3)
        k25 = gd['kp25'][t % len(gd['kp25'])].copy()
        if vid:
            k25[..., :2] += rng.uniform(-0.05, 0.05, size=k25[..., :2].shape).astype(np.float32)
        kp[:, :25] = torch.from_numpy(k25)
        out.append((s[t]['image'].cuda(), kp.cuda()))
    return out


def single_state(ad):
    return [ad.model.module.arena, ad.teacher.arena, ad.optimizer.m, ad.optimizer.v]


def tick(mv, inputs):
    """adapt_processed with per-stream entries (None: the stream sits the tick out)."""
    return mv.adapt_processed([None if x is None else x[0] for x in inputs], [None if x is None else x[1] for x in inputs])


def test_one_stream_is_the_webcam_adaptor(asset_dir, tmp_path, golden):
    gd = golden('adapt_webcam')
    n = gd['kp25'].shape[0]
    mv, ad = webcam_pool(tmp_path, gd, 1, 'mv'), single(tmp_path, gd, 'ad')
    for t, (img, kp) in enumerate(stream_inputs(gd, 0, n)):
        res = tick(mv, [(img, kp)])[0]
        ref = ad.adapt_processed(img, kp)
        assert mv.optim_step_record[0] == ad.optim_step_record and mv.video_steps[0] == ad.global_step == t + 1, t
        assert mv.feat_sims[0][t + 1] == ad.feat_sims[t + 1], t                      # keys follow WebcamAdaptor's
        for x, y in zip(state(mv, 0), single_state(ad)):
            assert torch.equal(x, y), t
        assert torch.equal(res['vts'], ref['vts']) and torch.equal(res['cam'], ref['cam']), t


def test_four_streams_follow_the_golden_and_their_own_runs(asset_dir, tmp_path, golden):
    from oracle.make_golden import sample_indices
    gd = golden('adapt_webcam')
    n = gd['kp25'].shape[0]
    mv = webcam_pool(tmp_path, gd, 4, 'mv')
    o = mv.options
    singles = {g: single(tmp_path, gd, f's{g}') for g in range(1, 4)}
    inputs = [stream_inputs(gd, g, n) for g in range(4)]
    names = [str(s) for s in gd['param_names']]
    lay = mv.base.model.module._lay
    n_outer = [0] * 4
    for t in range(n):
        res = tick(mv, [inputs[g][t] for g in range(4)])
        assert ('ul/motion_loss' in mv.fit_losses) == (t >= o.interval), t       # live one frame earlier than the benchmark's
        for g in range(4):
            trips = min(mv.optim_step_record[g][-1], o.optim_steps)
            n_outer[g] += 1 + trips
            bound = 4 * o.lr * n_outer[g]
            if g == 0:
                assert trips == int(gd['dyn_steps'][t]), t
                assert rel_err(res[0]['vts'][:, ::10], gd['verts_sub'][t]) < 1e-3 and rel_err(res[0]['cam'], gd['cam'][t]) < 1e-3, t
                views = dict(zip(lay.names, lay.views(mv.theta(0).clone())))
                for i, name in enumerate(names):
                    th = views[name].contiguous().flatten()[sample_indices(name, views[name].numel())].double().cpu().numpy()
                    assert np.abs(th - gd['theta_samples'][t][i]).max() <= bound, (t, name)
                continue
            ad = singles[g]
            ref = ad.adapt_processed(*inputs[g][t])
            assert mv.optim_step_record[g] == ad.optim_step_record, (g, t)
            assert rel_err(res[g]['vts'], ref['vts']) < 1e-3 and rel_err(res[g]['cam'], ref['cam']) < 1e-3, (g, t)
            assert float((mv.theta(g) - ad.model.module.arena).abs().max()) <= bound, (g, t)


def test_streams_that_drop_out(asset_dir, tmp_path, golden):
    """Stream X with None ticks: alone in slot 0 it follows a WebcamAdaptor fed only its frames; in slot 2 of a pool whose other
    slots run, pause and are started it is bit-identical to slot 0's run; an idle slot keeps every bit."""
    gd = golden('adapt_webcam')
    X, n = 5, 7
    xs = stream_inputs(gd, X, n)
    gaps = {2, 4}                                            # X's ticks with no person in view
    a = webcam_pool(tmp_path, gd, 4, 'a')
    ad = single(tmp_path, gd, 'ad')
    o = a.options
    traj_a, n_outer = [], 0
    for t in range(n):
        before = [state(a, g) for g in range(4)]
        res = tick(a, [None if t in gaps else xs[t], None, None, None])
        for g in range(1 if t not in gaps else 0, 4):
            assert all(torch.equal(x, y) for x, y in zip(before[g], state(a, g))), (t, g)
        if t in gaps:
            assert res == [None] * 4
            continue
        ref = ad.adapt_processed(*xs[t])
        n_outer += 1 + min(a.optim_step_record[0][-1], o.optim_steps)
        assert a.optim_step_record[0] == ad.optim_step_record and a.video_steps[0] == ad.global_step, t
        assert rel_err(res[0]['vts'], ref['vts']) < 1e-3 and rel_err(res[0]['cam'], ref['cam']) < 1e-3, t
        assert float((a.theta(0) - ad.model.module.arena).abs().max()) <= 4 * o.lr * n_outer, t
        traj_a.append(state(a, 0) + [res[0]['vts'].clone(), res[0]['cam'].clone()])
    del a, ad
    b = webcam_pool(tmp_path, gd, 4, 'b')
    others = {g: stream_inputs(gd, 10 + g, n + 3) for g in range(4)}
    traj_b = []
    for f in range(n + 3):
        if f == 3:
            b.start(2)                                       # X's camera replaces the stream slot 2 held
        if f == 5:
            b.start(3)
        t = f - 3
        x = None if f < 3 else (None if t in gaps else xs[t])
        ins = [others[0][f], None if f in (1, 4, 5) else others[1][f], x if f >= 3 else others[2][f],
               None if f in (2, 3, 4) else others[3][f]]
        idle = [g for g in range(4) if ins[g] is None]
        before = {g: state(b, g) for g in idle}
        res = tick(b, ins)
        for g in idle:
            assert all(torch.equal(p, q) for p, q in zip(before[g], state(b, g))), (f, g)
            assert res[g] is None
        if f >= 3 and t not in gaps:
            traj_b.append(state(b, 2) + [res[2]['vts'].clone(), res[2]['cam'].clone()])
    assert len(traj_a) == len(traj_b) == n - len(gaps)
    for i, (ra, rb) in enumerate(zip(traj_a, traj_b)):
        for name, x, y in zip(('theta', 'teacher', 'm', 'v', 'vts', 'cam'), ra, rb):
            assert torch.equal(x, y), (i, name)


def test_reload_keeps_history_and_frame_count(asset_dir, tmp_path, golden):
    gd = golden('adapt_webcam')
    n = 5
    mv = webcam_pool(tmp_path, gd, 2, 'mv')
    o = mv.options
    ad = single(tmp_path, gd, 'ad')
    ins = [stream_inputs(gd, 0, n), stream_inputs(gd, 1, n)]
    for t in range(3):
        tick(mv, [ins[0][t], ins[1][t]])
        ad.adapt_processed(*ins[0][t])
    other, hist = state(mv, 1), dict(mv.histories[0])
    mv.reload(0)
    base = mv.base
    assert torch.equal(mv.thetas[0], base.model.module.arena) and torch.equal(mv.teachers[0], base.teacher.arena)
    assert not mv.m[0].any() and not mv.v[0].any() and mv.step_counts[0] == 0
    assert mv.video_steps[0] == 3 and mv.histories[0].keys() == hist.keys()
    assert all(mv.histories[0][k][0] is hist[k][0] for k in hist)
    assert all(torch.equal(x, y) for x, y in zip(other, state(mv, 1)))
    # the reference's reload on the single-stream adaptor: model, teacher and Adam; history and step are kept
    ad.set_model_optim()
    ad.model.eval()
    ad.set_teacher()
    n_outer = 0
    for t in range(3, n):
        res = tick(mv, [ins[0][t], None])
        assert bool(torch.isfinite(mv.fit_losses['ul/motion_loss'][0])), t       # live right after the reload
        ref = ad.adapt_processed(*ins[0][t])
        n_outer += 1 + min(mv.optim_step_record[0][-1], o.optim_steps)
        assert mv.optim_step_record[0][-1] == ad.optim_step_record[-1] and mv.step_counts[0] == ad.optimizer.step_count, t
        assert rel_err(res[0]['vts'], ref['vts']) < 1e-3 and rel_err(res[0]['cam'], ref['cam']) < 1e-3, t
        assert float((mv.theta(0) - ad.model.module.arena).abs().max()) <= 4 * o.lr * n_outer, t
        assert all(torch.equal(x, y) for x, y in zip(other, state(mv, 1))), t


def raw_streams(n, seed):
    """Raw frames of three cameras (numpy uint8 1280x720, numpy float32 240x320, CUDA uint8 480x640) and detections."""
    rng = np.random.default_rng(seed)
    sizes = [(720, 1280), (240, 320), (480, 640)]
    out = []
    for t in range(n):
        frames, dets = [], []
        for g, (H, W) in enumerate(sizes):
            img = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
            frames.append(img if g == 0 else (img.astype(np.float32) if g == 1 else torch.from_numpy(img).cuda()))
            c = np.array([W / 2, H / 2]) + rng.uniform(-W / 8, W / 8, size=2)
            d = np.concatenate([c + rng.uniform(-H / 4, H / 4, size=(25, 2)), rng.uniform(0, 1, size=(25, 1))], 1)
            dets.append(d[None] if g != 1 else d)
        out.append((frames, dets))
    return out


def test_online_adaptation_end_to_end(asset_dir, tmp_path, golden):
    gd = golden('adapt_webcam')
    ticks = raw_streams(3, 9)
    ticks[1][0][2] = None                                    # camera 2 sees nobody at tick 1
    runs = []
    for r in range(2):
        mv = webcam_pool(tmp_path, gd, 3, f'r{r}', test_basemodel=1, dynamic_boa=0)
        outs = []
        for t, (frames, dets) in enumerate(ticks):
            res = mv.online_adaptation(frames, dets)
            outs.append(res)
            if r == 0 and t == 0:
                ad = single(tmp_path, gd, 'ad', test_basemodel=1, dynamic_boa=0)
                for g in range(3):
                    image, kp, bbox = ad.dataprocess(frames[g], np.asarray(dets[g]).reshape(25, 3), scaleFactor=1.2)
                    assert torch.equal(bits(mv._frames['image'][g:g + 1]), bits(image)), g
                    assert torch.equal(bits(mv._frames['smpl_j2d'][g:g + 1]), bits(kp)), g
                    assert np.array_equal(res[g]['bbox'], bbox), g
                    with torch.no_grad():
                        rot, shape, cam = ad.basemodel(image)
                        vts = ad.decode_smpl_params(rot, shape)['vts']
                    assert rel_err(res[g]['cam_base'], cam) < 1e-5 and rel_err(res[g]['vts_base'], vts) < 1e-5, g
                del ad
        assert outs[1][2] is None and mv.video_steps == [3, 3, 2]
        for res in outs:
            for g, x in enumerate(res):
                if x is None:
                    continue
                assert sorted(x) == ['bbox', 'cam', 'cam_base', 'vts', 'vts_base'], g
                assert x['vts'].shape == x['vts_base'].shape == (1, 6890, 3) and x['cam'].shape == x['cam_base'].shape == (1, 3)
                assert x['bbox'].shape == (1, 3) and torch.isfinite(x['vts']).all()
        assert not torch.equal(outs[-1][0]['vts'], outs[-1][0]['vts_base'])
        torch.cuda.synchronize()
        runs.append([[None if x is None else (x['vts'].clone(), x['cam'].clone()) for x in res] for res in outs] + [mv.thetas.clone()])
        del mv
    assert torch.equal(runs[0][-1], runs[1][-1])
    for ra, rb in zip(runs[0][:-1], runs[1][:-1]):
        for a, b in zip(ra, rb):
            assert (a is None) == (b is None) and (a is None or (torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])))
