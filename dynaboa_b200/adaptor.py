"""Benchmark driver on top of ``BaseAdaptor`` (the role of reference dynaboa_benchmark.py ``Adaptor``
:69-262: ``excute`` frame loop, ``adaptation`` bilevel + dynamic loop, ``inference`` metrics).

Two entry points per frame:

* ``adaptation(batch)``    -- the reference's control flow through torch autograd (``learner.adapt``,
  ``loss.backward()``, ``optimizer.step()``), every op a libdynaboa_b200 kernel.  This is the path the
  unchanged reference driver also exercises.
* ``adapt(batch)``         -- the same arithmetic without autograd: direct C-ABI calls into one flat gradient
  arena, Adam and the teacher EMA fused in one sweep, no host syncs except the ``dynamic_boa`` decision
  (see fused.py).  This is what ``bench.py`` times.
"""
import itertools
import os
import os.path as osp
import random

import numpy as np
import torch

from . import _lib, constants, hmr as hmr_mod, layout, state
from .base_adaptor import BaseAdaptor
from .fused import Frame, Step, _ArenaModel, fused_adapt

# DBOA_STEP_GRAPH=0 in the environment runs every frame of ``adapt`` eagerly (A/B measurements, debugging)
STEP_GRAPH = os.environ.get('DBOA_STEP_GRAPH', '1') != '0'


RESULT_FILES = ('lowerlevel_kp2dloss.pt', 'upperlevel_kp2dloss.pt', 'res.pt', 'lower_res.pt', 'steps_statistic_res.pt', 'feat_sims.pt',
                'optim_step_record.pt', 'res.txt')


def write_records(exppath, step, rec):
    """The eight result files of the reference driver, same names, same joblib pickles, same keys
    (dynaboa_benchmark.py:111-123), into the directory ``exppath``.  ``step``: the last frame's index, as ``res.txt`` reports
    it.  ``rec``: mpjpe, pampjpe, pve (one entry per frame), mpjpe_all_lower, pampjpe_all_lower (one list per inner step),
    mpjpe_statistics, pampjpe_statistics, feat_sims, optim_step_record, kp2dlosses_lower (a list) and kp2dlosses_upper (a dict
    by frame)."""
    import joblib
    p = lambda name: osp.join(exppath, name)
    mpjpe_all, pampjpe_all, pve_all = rec['mpjpe'], rec['pampjpe'], rec['pve']
    lower_m, lower_p = rec['mpjpe_all_lower'], rec['pampjpe_all_lower']
    joblib.dump({'kp2dloss': [float(x) for x in rec['kp2dlosses_lower']]}, p('lowerlevel_kp2dloss.pt'))
    joblib.dump({'kp2dloss': {k: float(v) for k, v in rec['kp2dlosses_upper'].items()}}, p('upperlevel_kp2dloss.pt'))
    joblib.dump({'mpjpe': mpjpe_all, 'pampjpe': pampjpe_all, 'pve': pve_all}, p('res.pt'))
    joblib.dump({'mpjpe': lower_m, 'pampjpe': lower_p}, p('lower_res.pt'))
    joblib.dump({'mpjpe': rec['mpjpe_statistics'], 'pampjpe': rec['pampjpe_statistics']}, p('steps_statistic_res.pt'))
    joblib.dump({'feat': rec['feat_sims']}, p('feat_sims.pt'))
    joblib.dump({'step': rec['optim_step_record']}, p('optim_step_record.pt'))
    with open(p('res.txt'), 'w') as f:
        f.write(f'Step:{step}: MPJPE:{np.mean(mpjpe_all)}, PAMPJPE:{np.mean(pampjpe_all)}, PVE:{np.mean(pve_all)}\n')
        for i in range(len(lower_m)):
            lo_m = np.mean(lower_m[i]) if len(lower_m[i]) else float('nan')
            lo_p = np.mean(lower_p[i]) if len(lower_p[i]) else float('nan')
            f.write(f'Lower-level  Step:{i} MPJPE:{lo_m}, PAMPJPE:{lo_p}\n')


class _StepGraph:
    """One single-video frame of ``fused_adapt`` captured as a CUDA graph: its static inputs (frame, keypoints, history frame),
    the graph, its records packed into one (n,) tensor and the number of library kernels it holds.  ``key``: the
    configuration it was captured in (``Adaptor._graph_key``)."""

    def __init__(self, key, image, kp):
        self.key, self.graph, self.launches = key, None, 0
        new = lambda t: torch.empty(t.shape, dtype=torch.float32, device=t.device)
        self.image, self.kp, self.hist_image, self.hist_kp = new(image), new(kp), new(image), new(kp)

    def pack(self, f):
        """Inside the capture: every record of the ``Frame`` f (one float each, G = 1) into ``packed``."""
        self.names, self.n_lower = list(f.fit), len(f.lower)
        self.packed = torch.cat([t.reshape(1) for t in [f.fit[k] for k in self.names] + list(f.lower) + [f.upper_loss]])

    def frame(self):
        """The ``Frame`` of the last replay, from a copy of ``packed``: the next replay does not change it."""
        p, n = self.packed.clone(), len(self.names)
        f = Frame(1)
        f.fit = {k: p[i:i + 1] for i, k in enumerate(self.names)}
        f.lower = [p[n + i:n + i + 1] for i in range(self.n_lower)]
        f.upper_loss = p[-1:]
        return f


class Adaptor(BaseAdaptor):
    kp_range = (25, 24)          # joints of the 2D and motion terms (fused.Step)
    motion_lead = 0              # the motion term is live while global_step + motion_lead - interval > 0 (before save_hist)
    step_graph = True            # adapt may replay its steady-state frame as a CUDA graph (see _graph_key)
    # the records a saved state carries (save_state)
    RECORDS = ('feat_sims', 'optim_step_record', 'mpjpe_statistics', 'pampjpe_statistics', 'mpjpe_all_lower', 'pampjpe_all_lower',
               'kp2dlosses_lower', 'kp2dlosses_upper', 'last_upper_loss', 'last_retrieval', 'optimized_step')

    def __init__(self, options):
        super().__init__(options)
        self.model.eval()        # the reference driver does this before every frame (dynaboa_benchmark.py:89)
        self.reset_records()
        self.fused_eval = 'final'                          # adapt's evaluations: 'none', 'final' or 'all'
        self.phase_events = None                           # a list: adapt records CUDA events at its phase boundaries
        self._graph, self._graph_warm = None, None         # adapt's captured frame; the key of the last eager frame
        self._weights_read = None                          # recorded by predict_async after its read of the weights

    def reset_records(self):
        n = len(self.dataloader)
        self.feat_sims, self.optim_step_record = {}, []
        self.mpjpe_statistics, self.pampjpe_statistics = [[] for _ in range(n)], [[] for _ in range(n)]
        self.mpjpe_all_lower = [[] for _ in range(self.options.inner_step)]
        self.pampjpe_all_lower = [[] for _ in range(self.options.inner_step)]
        self.history, self.kp2dlosses_lower, self.kp2dlosses_upper = {}, [], {}

    # ------------------------------------------------------------------ frame loop (reference :71-123)
    def excute(self, max_frames=None, fused=False, checkpoint=None, every=0):
        """The frame loop.  ``checkpoint``: a video-state file (``save_state``); when it exists the run resumes from it, skipping
        the frames it already adapted, and with ``every`` > 0 it is written after every ``every`` frames.  A resumed run
        writes the same eight result files, byte for byte, as one that was never interrupted."""
        self.reset_records()
        mpjpe_all, pampjpe_all, pve_all = [], [], []
        start = 0
        if checkpoint is not None and osp.exists(checkpoint):
            run = self.load_state(checkpoint)
            start, mpjpe_all, pampjpe_all, pve_all = run['next_frame'], run['mpjpe'], run['pampjpe'], run['pve']
        for step, batch in enumerate(self._batches_from(start), start):
            if max_frames is not None and step >= max_frames:
                break
            self.global_step, self.fit_losses = step, {}
            batch = {k: v.to(self.device) if isinstance(v, torch.Tensor) else v for k, v in batch.items()}
            self.model.eval()
            mpjpe, pampjpe, pve = (self.adapt(batch) if fused else self.adaptation(batch))
            self.fit_losses.update({'metrics/mpjpe': mpjpe, 'metrics/pampjpe': pampjpe, 'metrics/pve': pve})
            self.write_summaries(self.fit_losses)
            mpjpe_all.append(mpjpe); pampjpe_all.append(pampjpe); pve_all.append(pve)
            if checkpoint is not None and every and (step + 1) % every == 0:
                self.save_state(checkpoint, run=dict(next_frame=step + 1, mpjpe=mpjpe_all, pampjpe=pampjpe_all, pve=pve_all))
        summary = dict(mpjpe=float(np.mean(mpjpe_all)), pampjpe=float(np.mean(pampjpe_all)), pve=float(np.mean(pve_all)))
        self.save_records(mpjpe_all, pampjpe_all, pve_all)
        return summary

    def _batches_from(self, start):
        """The batches of ``dataloader`` from batch ``start`` on: a ``DataLoader`` over an indexable dataset skips the first
        ``start`` batches without loading them; any other iterable is advanced with ``itertools.islice``."""
        dl = self.dataloader
        if start == 0:
            return dl
        ds = getattr(dl, 'dataset', None)
        if isinstance(dl, torch.utils.data.DataLoader) and hasattr(ds, '__len__') and dl.batch_size is not None:
            rest = torch.utils.data.Subset(ds, range(min(start * dl.batch_size, len(ds)), len(ds)))
            return torch.utils.data.DataLoader(rest, batch_size=dl.batch_size, shuffle=False, num_workers=0, collate_fn=dl.collate_fn,
                                               drop_last=dl.drop_last)
        return itertools.islice(dl, start, None)

    def save_records(self, mpjpe_all, pampjpe_all, pve_all):
        """The eight result files of the reference driver (``write_records``)."""
        write_records(self.exppath, self.global_step, dict(
            mpjpe=mpjpe_all, pampjpe=pampjpe_all, pve=pve_all, mpjpe_all_lower=self.mpjpe_all_lower, pampjpe_all_lower=self.pampjpe_all_lower,
            mpjpe_statistics=self.mpjpe_statistics, pampjpe_statistics=self.pampjpe_statistics, feat_sims=self.feat_sims,
            optim_step_record=self.optim_step_record, kp2dlosses_lower=self.kp2dlosses_lower, kp2dlosses_upper=self.kp2dlosses_upper))

    def _outer_step(self, loss):
        self.optimizer.zero_grad()
        loss.backward()
        self.optimizer.step()
        if self.options.use_meanteacher:
            self.update_teacher(self.teacher, self.model)

    # ------------------------------------------------------------------ bilevel step through autograd (reference :126-201)
    def adaptation(self, batch):
        o = self.options
        image, kp = batch['image'], batch['smpl_j2d']
        self.save_hist(image, kp)
        if not o.use_boa:
            loss, _ = self.lower_level_adaptation(image, kp, None, self.model)
            self.optimizer.zero_grad(); loss.backward(); self.optimizer.step()
            return self.inference(batch, self.model)

        with torch.no_grad():
            init_features = self.model(image, need_feature=True)[3]
        learner = self.model.clone()
        for i in range(o.inner_step):
            lower_loss, _ = self.lower_level_adaptation(image, kp, None, learner)
            learner.adapt(lower_loss)
            mpjpe, pampjpe, _ = self.inference(batch, learner)
            self.fit_losses[f'metrics/lower_{i}_mpjpe'], self.fit_losses[f'metrics/lower_{i}_pampjpe'] = mpjpe, pampjpe
            self.mpjpe_all_lower[i].append(mpjpe); self.pampjpe_all_lower[i].append(pampjpe)
        upper_loss, _ = self.upper_level_adaptation(image, kp, None, learner)
        self.last_upper_loss = upper_loss.detach()
        self._outer_step(upper_loss)
        mpjpe, pampjpe, pve = self.inference(batch, self.model)
        if self.global_step < len(self.mpjpe_statistics):
            self.mpjpe_statistics[self.global_step], self.pampjpe_statistics[self.global_step] = [mpjpe], [pampjpe]

        if o.dynamic_boa:
            with torch.no_grad():
                adapted = self.model(image, need_feature=True)[3]
                sims = self.cal_feature_diff(init_features, adapted)
            self.feat_sims[self.global_step] = [sims]
            self.optimized_step = 0
            while 1 - sims[12]['cos'] > o.cos_sim_threshold:
                self.optimized_step += 1
                if self.optimized_step > o.optim_steps:
                    break
                upper_loss, adapted = self.upper_level_adaptation(image, kp, None, self.model)
                self._outer_step(upper_loss)
                with torch.no_grad():
                    init_features = adapted
                    adapted = self.model(image, need_feature=True)[3]
                    sims = self.cal_feature_diff(init_features, adapted)
                self.feat_sims[self.global_step].append(sims)
                mpjpe, pampjpe, pve = self.inference(batch, self.model)
            self.optim_step_record.append(self.optimized_step)
        return mpjpe, pampjpe, pve

    # ------------------------------------------------------------------ saved state (state.py, DESIGN.md section 11)
    def _check_state_support(self):
        opt = self.optimizer
        if opt.grad_sync is not None or opt.pre_step_hook is not None:
            raise ValueError('the state of a data-parallel (dist.attach) optimizer cannot be saved or loaded: its ranks would have '
                             'to be resumed together')

    def save_state(self, path, run=None):
        """Write this video's state to ``path`` (``state.video_state``, atomically): theta, teacher, Adam moments and step count,
        ``global_step``, the history ring, the ``random``, torch CPU and torch CUDA generator states and every record
        (``run``: ``excute``'s own, kept with them).  Call it between frames: the copies to the host wait for the frame's last
        write to the arenas on the current stream."""
        self._check_state_support()
        model, opt = getattr(self.model, 'module', self.model), self.optimizer
        records = {k: getattr(self, k, None) for k in self.RECORDS}
        records['run'] = run
        st = state.video_state(self.options, 'adaptor', 1, model.arena, self.teacher.arena if self.options.use_meanteacher else None,
                               opt.m, opt.v, opt.step_count, self.global_step,
                               [(k, h['image'], h['s2d']) for k, h in sorted(self.history.items())],
                               dict(random=random.getstate(), torch=torch.get_rng_state(), cuda=torch.cuda.get_rng_state(self.device)),
                               records)
        state.write(path, st)

    def load_state(self, path):
        """Continue from the state ``save_state`` wrote to ``path``: every check runs before any device work (ValueError), then
        the arenas, moments and generator states are restored in place and the records replaced.  The next frame of ``adapt``
        runs eagerly and the one after is captured again.  Returns the ``run`` the state was saved with."""
        self._check_state_support()
        st = state.read_video(path, self.options, 'adaptor')
        model, opt = getattr(self.model, 'module', self.model), self.optimizer
        torch.cuda.synchronize(self.device)                # no reader of the weights (predict_async) is still in flight
        model.arena.copy_(st['theta'])
        if self.options.use_meanteacher:
            self.teacher.arena.copy_(st['teacher'])
        opt.m.copy_(st['m'])
        opt.v.copy_(st['v'])
        opt.step_count, opt.wait_before_write = st['step_count'], []
        self.global_step = st['frames']
        self.history = {k: {'image': a.to(self.device), 's2d': b.to(self.device)} for k, (a, b) in st['history'].items()}
        rng = st['rng']
        random.setstate(rng['random'])
        torch.set_rng_state(rng['torch'])
        torch.cuda.set_rng_state(rng['cuda'], self.device)
        rec = st['records']
        for k in self.RECORDS:
            v = rec.get(k)
            setattr(self, k, v.to(self.device) if isinstance(v, torch.Tensor) and k == 'last_upper_loss' else v)
        self._graph, self._graph_warm = None, None
        torch.cuda.synchronize(self.device)
        return rec.get('run')

    def export_model(self, path):
        """Write the adapted weights as a checkpoint in the reference's format, ``{'model': {'module.' + name: tensor}}`` with
        the ``init_*`` buffers: it loads as ``model_file`` (and into the reference's ``hmr()``)."""
        model = getattr(self.model, 'module', self.model)
        state.write(path, {'model': layout.state_dict(model.arena, model._buffers, prefix='module.')})

    # ------------------------------------------------------------------ evaluation (reference :204-262)
    def predict(self, image, model=None):
        """rotmat, betas, cam, joints49, vertices for ``image`` (no adaptation)."""
        model = self.model if model is None else model
        with torch.no_grad():
            rot, shape, cam = model(image)
            out = self.decode_smpl_params(rot, shape)
        return dict(rotmat=rot, betas=shape, cam=cam, joints=out['s3d'], vertices=out['vts'])

    def predict_async(self, image):
        """``predict`` issued on a side stream.  The output forward of frame t and the adaptation of frame t+1 read the
        same weights, so the caller can go on enqueueing the next frame on its own stream: the two chains of small kernels
        overlap on the device, and the next optimiser step waits for this read before it overwrites the weights.
        Returns (outputs, event); consumers on another stream (or the host) wait for the event first."""
        cur = torch.cuda.current_stream()
        if getattr(self, 'output_stream', None) is None:
            self.output_stream = torch.cuda.Stream(device=image.device)
        side = self.output_stream
        side.wait_stream(cur)                              # the weights (and the frame) are ready
        with torch.cuda.stream(side):
            out = self.predict(image)
            ev = torch.cuda.Event()
            ev.record(side)
            if self._weights_read is None:
                self._weights_read = torch.cuda.Event()
            self._weights_read.record(side)                # what a captured optimiser step waits for (external wait)
        image.record_stream(side)
        for v in out.values():                             # allocated on the side stream, read by the caller's stream after the event
            v.record_stream(cur)
        self.optimizer.wait_before_write.append(ev)
        return out, ev

    def inference(self, batch, model, need_feature=False):
        image = batch['image']
        model.eval()
        with torch.no_grad():
            out = model(image, need_feature)
            pred_rotmat, pred_shape, pred_cam = out[0], out[1], out[2]
            pred_vertices = self.decode_smpl_params(pred_rotmat, pred_shape)['vts']
            gt_vertices, gt_neutral = self._gt_meshes(batch)
            # H36M-regressor joints, MPJPE, Procrustes PA-MPJPE and PVE in two launches; ONE 3-float read-back per sample
            # (the reference copies joints and both meshes to the host and runs a numpy SVD per sample: :217-240)
            metrics = self.eval_metrics(pred_vertices, gt_vertices, gt_neutral).cpu().numpy()
            mpjpe, pampjpe, pve = metrics[:, 0], metrics[:, 1], float(metrics[:, 2].mean())
        if getattr(self.options, 'cache_results', 1):        # the reference always dumps Pred_<step>.pt (:250-254); 0 turns the disk write off
            cam_t = torch.stack([pred_cam[:, 1], pred_cam[:, 2], 2 * 5000. / (constants.IMG_RES * pred_cam[:, 0] + 1e-9)], dim=-1)
            import joblib
            joblib.dump({'verts': pred_vertices.cpu().numpy(), 'cam': cam_t.cpu().numpy(), 'rotmat': pred_rotmat.cpu().numpy(),
                         'beta': pred_shape.cpu().numpy()}, osp.join(self.exppath, 'result', f'Pred_{self.global_step}.pt'))
        if need_feature:
            return mpjpe * 1000, pampjpe * 1000, pve * 1000, out[3]
        return mpjpe * 1000, pampjpe * 1000, pve * 1000

    def eval_metrics(self, pred_vertices, gt_vertices, gt_vertices_neutral, groups=1, active=None):
        """(B,3) device tensor: MPJPE, PA-MPJPE, PVE (metres) of each sample -- ``dboa_eval_metrics_active``.  ``groups``
        videos of B / groups rows each, of which only those whose bit is set in ``active`` (an int; None: all) are evaluated:
        the rows of the others are left unwritten."""
        B, dev = pred_vertices.shape[0], pred_vertices.device
        if getattr(self, '_eval_consts', None) is None or self._eval_consts[0].device != dev:
            self._eval_consts = (self.J_regressor.to(dev).contiguous().float(),
                                 torch.as_tensor(np.asarray(self.joint_mapper_h36m), dtype=torch.int32, device=dev))
        J, jmap = self._eval_consts
        _lib.require_cuda(pred_vertices, gt_vertices, gt_vertices_neutral)
        scratch = torch.empty(_lib.load().dboa_eval_scratch_floats(B, J.shape[0]), dtype=torch.float32, device=dev)
        out = torch.empty(B, 3, dtype=torch.float32, device=dev)
        keep = [t.contiguous().float() for t in (pred_vertices, gt_vertices, gt_vertices_neutral)]
        args = (_lib.ptr(keep[0]), _lib.ptr(keep[1]), _lib.ptr(keep[2]), _lib.ptr(J), int(J.shape[0]), int(pred_vertices.shape[1]), _lib.ptr(jmap),
                int(jmap.numel()), _lib.ptr(scratch), _lib.ptr(out), B)
        _lib.call('dboa_eval_metrics_active', *args, int(groups), (1 << int(groups)) - 1 if active is None else int(active), _lib.stream())
        return out

    def _gt_meshes(self, batch):
        """The ground-truth meshes of ``batch``: gender-selected (male / female SMPL) and neutral."""
        pose, betas = batch['pose'], batch['betas']
        gt = self.smpl_male(global_orient=pose[:, :3], body_pose=pose[:, 3:], betas=betas).vertices
        gt_f = self.smpl_female(global_orient=pose[:, :3], body_pose=pose[:, 3:], betas=betas).vertices
        gt = torch.where((batch['gender'] == 1).view(-1, 1, 1), gt_f, gt)
        return gt, self.smpl_neutral(betas=betas, body_pose=pose[:, 3:], global_orient=pose[:, :3], pose2rot=True).vertices

    # ------------------------------------------------------------------ the same step without autograd (fused.py)
    def adapt(self, batch):
        """One frame through ``fused.fused_adapt``, its records filed under the reference's names; returns ``inference``'s.

        In the steady state of a single video (``_graph_key``) the frame is captured once as a CUDA graph, after one eager
        frame in the same configuration, and replayed from then on: same kernels, grids and order, so every result is the
        eager frame's, bit for bit, without the host-side cost of enqueueing some 800 launches."""
        import torch.distributed as dist
        key = self._graph_key(batch)
        if key is not None and self._graph is not None and self._graph.key == key:
            return self._file(self._replay(batch))
        if key is not None and self._graph_warm == key:
            return self._file(self._capture(batch, key))
        s, opt = self._step or self._make_step(), self.optimizer
        s.eval_mode, s.phase_events = self.fused_eval, self.phase_events
        s.grad_sync = opt.grad_sync if (opt.grad_sync is not None and dist.is_initialized() and dist.get_world_size() > 1) else None
        f = fused_adapt(s, batch, 1, [self.global_step])
        self._graph_warm = key
        return self._file(f)

    def _file(self, f):
        self.fit_losses.update({k: v[0] for k, v in f.fit.items()})
        self.kp2dlosses_lower += [v[0] for v in f.lower]
        if 'ul/s2dloss' in f.fit:
            self.kp2dlosses_upper[self.global_step] = f.fit['ul/s2dloss'][0]
        self.last_upper_loss = f.upper_loss[0]
        if f.picks is not None:
            self.last_retrieval = f.picks[0]
        if f.steps is not None:
            self.feat_sims[self.global_step], self.optimized_step = f.sims[0], f.steps[0]
            self.optim_step_record.append(f.steps[0])
        return f.result

    # ------------------------------------------------------------------ the frame as a CUDA graph
    def _graph_key(self, batch):
        """The configuration a captured frame of ``batch`` is valid in, or None when the frame runs eagerly.  A graph needs a
        frame whose every host-side decision is fixed: one video on one GPU, no retrieval (its cluster index goes through the
        host), no dynamic loop (its trip count does), no evaluation, the motion term live, the teacher's dropout from torch's
        generator (a replay draws as an eager frame does), the default network plan; and the same tensors as at capture."""
        o, opt = self.options, self.optimizer
        if not (STEP_GRAPH and self.step_graph and o.use_boa) or o.retrieval or o.dynamic_boa or self.fused_eval != 'none':
            return None
        if self.phase_events is not None or opt.grad_sync is not None or opt.pre_step_hook is not None:
            return None
        if self.global_step + self.motion_lead - o.interval <= 0:
            return None
        masked = False
        if o.use_meanteacher:
            if self.teacher.mask_provider is not None or hmr_mod.DEFAULT_MASK_PROVIDER is not None:
                return None
            masked = self.teacher.training
        lib = _lib.load()
        if lib.dboa_get_fused_forward() or lib.dboa_get_fused_backward():
            return None
        s = self._step or self._make_step()
        image, kp = batch['image'], batch['smpl_j2d']
        arenas = (s.theta, s.grad, s.teacher, opt.m, opt.v)
        return (id(s), tuple(None if t is None else t.data_ptr() for t in arenas), masked, tuple(image.shape), image.device,
                tuple(kp.shape))

    def _graph_prologue(self, g, batch):
        """What a replayed frame takes from the host: the frame and its keypoints, the history (saved here, as ``fused_adapt``
        saves it) and the step's Adam scalars.  The graph waits for ``predict_async``'s reads through ``_weights_read``."""
        g.image.copy_(batch['image'])
        g.kp.copy_(batch['smpl_j2d'])
        self.save_hist(g.image, g.kp)
        hist_image, hist_kp = self.get_hist()
        g.hist_image.copy_(hist_image)
        g.hist_kp.copy_(hist_kp)
        self.optimizer.write_scalars(self.options.alpha)
        self.optimizer.wait_before_write = []

    def _capture(self, batch, key):
        s, lib = self._step, _lib.load()
        _lib.check(lib.dboa_prepare_graph(), 'dboa_prepare_graph')
        if self._weights_read is None:                     # the captured wait needs an event; recorded once, it is a no-op
            self._weights_read = torch.cuda.Event()
            self._weights_read.record()
        g = _StepGraph(key, batch['image'], batch['smpl_j2d'])
        self._graph_prologue(g, batch)
        s.eval_mode, s.phase_events, s.grad_sync = 'none', None, None
        hooks = s.save_hist, s.get_hist, s.adam
        s.save_hist = lambda image, kp, mask: None
        s.get_hist = lambda live: (g.hist_image, g.hist_kp)
        s.adam = lambda mask, teacher=None, alpha=0.0: self.optimizer.step_captured(
            self._weights_read, teacher=None if teacher is None else self.teacher)
        graph = torch.cuda.CUDAGraph()
        n0 = lib.dboa_launch_count()
        try:
            with torch.cuda.graph(graph, capture_error_mode='thread_local'):
                g.pack(fused_adapt(s, {'image': g.image, 'smpl_j2d': g.kp}, 1, [self.global_step]))
        finally:
            s.save_hist, s.get_hist, s.adam = hooks
        g.graph, g.launches = graph, lib.dboa_launch_count() - n0
        self._graph = g
        graph.replay()                                     # this frame: its kernels were counted as they were captured
        return g.frame()

    def _replay(self, batch):
        g = self._graph
        self._graph_prologue(g, batch)
        g.graph.replay()
        _lib.call('dboa_launch_credit', g.launches)
        return g.frame()

    def _make_step(self):
        o = self.options
        model = getattr(self.model, 'module', self.model)
        teacher = self.teacher if o.use_meanteacher else None
        self._step = Step(o, 1, model.arena, model.grad_arena(), model._buffers, self.smpl_neutral, self.gmm_f,
                          teacher=None if teacher is None else teacher.arena, teacher_buffers=None if teacher is None else teacher._buffers,
                          teacher_masks=None if teacher is None else lambda B, device, mask: teacher._masks(B, device),
                          kp_range=self.kp_range, motion_lead=self.motion_lead, bank=self.bank if o.retrieval else None,
                          rngs=[random] if o.retrieval else None, save_hist=lambda image, kp, mask: self.save_hist(image, kp),
                          get_hist=lambda live: self.get_hist(), adam=self._adam, evaluate=self._evaluate, reduce_terms=self._reduce_terms)
        return self._step

    def _adam(self, mask, teacher=None, alpha=0.0):
        if self._step.grad_sync is not None:
            self.optimizer.reduced = True                  # the level's last backward all-reduces on the communication stream
        self.optimizer.step(teacher=None if teacher is None else self.teacher, alpha=alpha)

    def _evaluate(self, batch, arena, mask, inner):
        return self.inference(batch, self.model if inner is None else _ArenaModel(getattr(self.model, 'module', self.model), arena))


class InternetAdaptor(Adaptor):
    """Client of the same path without ground truth (reference dynaboa_internet.py ``Adaptor`` :68-168): the adaptation is
    ``Adaptor.adaptation`` minus the per-step evaluation, ``inference`` only decodes the mesh and caches ``Pred_<step>.pt``."""

    def reset_records(self):
        super().reset_records()
        self.mpjpe_statistics, self.pampjpe_statistics = [], []

    def excute(self, max_frames=None, fused=False):
        self.reset_records()
        outs = []
        for step, batch in enumerate(self.dataloader):
            if max_frames is not None and step >= max_frames:
                break
            self.global_step, self.fit_losses = step, {}
            batch = {k: v.to(self.device) if isinstance(v, torch.Tensor) else v for k, v in batch.items()}
            self.model.eval()
            if fused:
                self.fused_eval = 'none'
                self.adapt(batch)
            else:
                self.adaptation(batch)
            outs.append(self.inference(batch, self.model))
        return outs

    def inference(self, batch, model, need_feature=False):
        """reference dynaboa_internet.py:142-168: no metrics (there is no ground truth), cached predictions only."""
        model.eval()
        with torch.no_grad():
            out = model(batch['image'], need_feature)
            pred_rotmat, pred_shape, pred_cam = out[0], out[1], out[2]
            pred_vertices = self.decode_smpl_params(pred_rotmat, pred_shape)['vts']
        cam_t = torch.stack([pred_cam[:, 1], pred_cam[:, 2], 2 * 5000. / (constants.IMG_RES * pred_cam[:, 0] + 1e-9)], dim=-1)
        res = {'verts': pred_vertices, 'cam': cam_t, 'rotmat': pred_rotmat, 'beta': pred_shape}
        if getattr(self.options, 'cache_results', 1):
            import joblib
            joblib.dump({k: v.cpu().numpy() for k, v in res.items()}, osp.join(self.exppath, 'result', f'Pred_{self.global_step}.pt'))
        zero = np.zeros(pred_rotmat.shape[0], np.float32)
        return (zero, zero, 0.0, out[3]) if need_feature else (zero, zero, 0.0)
