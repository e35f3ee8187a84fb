"""Adaptation runtime on the CUDA library (drop-in for reference base_adaptor.py ``BaseAdaptor`` :36-447).

Same constructor argument (the argparse namespace of the drivers), same attributes and method names as the
reference, so the unchanged ``dynaboa_benchmark.Adaptor`` subclass runs on top of it; every tensor operation
goes through libdynaboa_b200 (HMR forward/backward, SMPL, projection, fused loss heads, fused Adam / EMA,
one-launch feature test, nearest-centre retrieval).  Deliberate departures from the reference, all
behaviour-preserving (SURVEY.md Appendix D):

* history frames stay on the device and are pruned after ``interval`` steps (reference: unbounded host dict);
* retrieval gathers rows of a device-resident exemplar bank (reference: JPEG reads through ``SourceDataset``),
  concatenating tensor fields for any ``sample_num`` (the reference's loop only works for 1);
* ``cal_feature_diff`` syncs once instead of 15 times; the averaged value keeps the reference's ``/ 14``.
"""
import os
import os.path as osp
import random

import numpy as np
import torch

from . import config, constants, losses, optim
from .fused import Bank, cosines, retrieve
from .geometry import batch_rodrigues, project_normalized
from .hmr import hmr
from .maml import MAML
from .prior import MaxMixturePrior
from .smpl import SMPL
from . import _lib


class _NullWriter:
    def add_scalar(self, *a, **k):
        pass


class BaseAdaptor:
    def __init__(self, options):
        self.options = options
        self.exppath = osp.join(options.expdir, options.expname)
        for sub in ('mesh', 'image', 'result'):
            os.makedirs(osp.join(self.exppath, sub), exist_ok=True)
        if getattr(options, 'tensorboard', 1):
            from torch.utils.tensorboard import SummaryWriter
            self.summary_writer = SummaryWriter(self.exppath)
        else:
            self.summary_writer = _NullWriter()
        if not torch.cuda.is_available():
            raise RuntimeError('dynaboa_b200 needs a CUDA device (sm_90a); there is no CPU path')
        self.device = torch.device('cuda', torch.cuda.current_device())
        _lib.load()
        self.seed_everything(options.seed)
        options.mixtrain = options.lower_level_mixtrain or options.upper_level_mixtrain
        if options.mixtrain and not options.retrieval:
            raise ValueError('mixtrain needs retrieval=1 (the reference dereferences None here, base_adaptor.py:347)')
        if options.retrieval:
            self.load_h36_cluster_res()
        self.set_model_optim()
        if options.use_meanteacher:
            self.set_teacher()
        self.set_dataloader()
        self.set_criterion()
        self.setup_smpl()
        self.history, self.fit_losses, self.global_step = {}, {}, 0
        self.kp2dlosses_lower, self.kp2dlosses_upper = [], {}
        self._cos_partial = None                     # scratch of the feature test, sized from the features on first use
        self.dp_group = None                         # torch.distributed group of the data-parallel ranks (None: default group)

    # ------------------------------------------------------------------ set-up (reference :70-158)
    def seed_everything(self, seed):
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        torch.cuda.manual_seed_all(seed)

    def load_h36_cluster_res(self):
        cl = torch.load(config.RETRIEVAL_CLUSTERS, weights_only=False)
        self.centers = torch.as_tensor(np.asarray(cl['centers'])).float().to(self.device).contiguous()
        self.index = cl['index']
        bank = torch.load(config.RETRIEVAL_BANK, weights_only=False)
        self.h36m_bank = {k: v.float().to(self.device).contiguous() for k, v in bank.items()}
        self.bank = Bank(self.centers, self.index, self.h36m_bank, torch.zeros(self.centers.shape[0], dtype=torch.float32, device=self.device))
        self._best = torch.zeros(1, dtype=torch.int32, device=self.device)

    def get_h36m_data(self, indice):
        return {k: v[indice:indice + 1] for k, v in self.h36m_bank.items()}

    def retrieval(self, feature):
        """reference :82-96: nearest cluster centre by cosine distance, then ``random.sample`` inside it."""
        (self.last_retrieval,), batch = retrieve(self.bank, feature.detach().reshape(1, -1)[:, :2048], [random], 1, self._best,
                                                 self.options.sample_num)
        return batch

    def set_model_optim(self):
        checkpoint = torch.load(self.options.model_file, map_location='cpu', weights_only=False)
        model = hmr(config.SMPL_MEAN_PARAMS)
        if self.options.use_boa:
            self.model = MAML(model, lr=self.options.fastlr, first_order=True).to(self.device)
            self.model.load_state_dict(checkpoint['model'], strict=True)
        else:
            self.model = model.to(self.device)
            self.model.load_state_dict({k.replace('module.', ''): v for k, v in checkpoint['model'].items()}, strict=True)
        self.optimizer = optim.FusedAdam(self.model.parameters(), lr=self.options.lr, betas=(self.options.beta1, self.options.beta2),
                                         model=self.model)
        self._step = None                    # Adaptor.adapt's fused.Step: built again over the new arenas

    def set_teacher(self):
        checkpoint = torch.load(self.options.model_file, map_location='cpu', weights_only=False)
        model = hmr(config.SMPL_MEAN_PARAMS)
        for p in model.parameters():
            p.requires_grad_(False)
        self.teacher = model.to(self.device)
        self.teacher.load_state_dict({k.replace('module.', ''): v for k, v in checkpoint['model'].items()}, strict=True)
        self._step = None
        # the reference never calls teacher.eval(): its dropout stays active (SURVEY.md Appendix D)
        if not getattr(self.options, 'teacher_dropout', 1):
            self.teacher.eval()

    def set_dataloader(self):
        from torch.utils.data import DataLoader
        from .datasets import PW3D, Internet_dataset
        if self.options.dataset == '3dpw':
            dataset, self.imgdir = PW3D(self.options), config.PW3D_ROOT
        else:
            dataset = Internet_dataset(self.options)
            self.imgdir = getattr(dataset, 'imgdir', osp.join(config.InternetData_ROOT, 'images'))   # DYNABOA_INTERNET_ROOT applies
        self.dataloader = DataLoader(dataset, batch_size=self.options.batch_size, shuffle=False, num_workers=0)

    def set_criterion(self):
        self.gmm_f = MaxMixturePrior(prior_folder=getattr(self.options, 'prior_folder', None), num_gaussians=8,
                                     dtype=torch.float32).to(self.device)

    def setup_smpl(self):
        self.smpl_neutral = SMPL(config.SMPL_MODEL_DIR, create_transl=False).to(self.device)
        self.smpl_male = SMPL(config.SMPL_MODEL_DIR, gender='male', create_transl=False).to(self.device)
        self.smpl_female = SMPL(config.SMPL_MODEL_DIR, gender='female', create_transl=False).to(self.device)
        self.joint_mapper_h36m = constants.H36M_TO_J14
        self.joint_mapper_gt = constants.J24_TO_J14
        self.J_regressor = torch.from_numpy(np.load(config.JOINT_REGRESSOR_H36M)).float()

    # ------------------------------------------------------------------ small pieces (reference :160-219)
    def projection(self, cam, s3d, eps=1e-9):
        normed = project_normalized(cam, s3d)
        return {'ori': normed * (constants.IMG_RES / 2.0), 'normed': normed}

    def save_hist(self, image, s2d):
        self.history[self.global_step] = {'image': image.detach().clone(), 's2d': s2d.detach().clone()}
        stale = self.global_step - self.options.interval - 1
        if stale in self.history:
            del self.history[stale]

    def get_hist(self):
        h = self.history[self.global_step - self.options.interval]
        image, s2d = h['image'], h['s2d']
        if isinstance(image, np.ndarray):
            image, s2d = torch.from_numpy(image), torch.from_numpy(s2d)
        return image.to(self.device), s2d.to(self.device)

    def decode_smpl_params(self, poses, beta, gender='neutral', pose2rot=False):
        smpl = {'neutral': self.smpl_neutral, 'male': self.smpl_male, 'female': self.smpl_female}[gender]
        out = smpl(betas=beta, body_pose=poses[:, 1:], global_orient=poses[:, 0].unsqueeze(1), pose2rot=pose2rot)
        return {'s3d': out.joints, 'vts': out.vertices}

    def update_teacher(self, teacher, model):
        optim.ema_update(teacher, model, self.options.alpha)

    def excute(self):
        pass

    def adaptation(self):
        pass

    def cal_feature_diff(self, features_i, features_j):
        """reference :211-219: the cosine of each feature pair, one video of ``fused.cosines`` (the sums all-reduced over the
        data-parallel ranks first: ``_reduce_terms``)."""
        cos, self._cos_partial = cosines(features_i, features_j, 1, 1, self._cos_partial, self._reduce_terms)
        cos, n = cos[0], len(features_i)
        self.fit_losses['feat_sim/cos_sim'] = cos.sum() / (n - 1)        # reference :218 divides by the last index
        return {i: {'cos': float(cos[i])} for i in range(n)}

    def _reduce_terms(self, terms):
        """Data parallel: the feature test's sums all-reduced over the ranks (the reference flattens across the batch, :215), so
        every rank takes the same dynamic steps -- the gradient all-reduce inside them would dead-lock otherwise."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self.dp_group) > 1:
            dist.all_reduce(terms, op=dist.ReduceOp.SUM, group=self.dp_group)

    # ------------------------------------------------------------------ losses (reference :320-422)
    def cal_shape_prior(self, pred_betas):
        return self._single_term(1, beta=pred_betas)

    def cal_pose_prior(self, pred_rotmat, betas):
        return self.gmm_f.from_rotmat(pred_rotmat).mean()

    def _single_term(self, which, beta=None):
        B = beta.shape[0]
        z = lambda *s: torch.zeros(*s, device=beta.device)
        w = [0.0] * 8
        w[which] = 1.0
        total, _ = losses.loss_multi(z(B, 49, 2), z(B, 49, 3), z(B, 24, 3, 3), beta, w)
        return total

    def cal_s3d_loss(self, pred_s3d, gt_s3d, conf):
        """Hip-centred masked MSE (reference :412-422); inputs (N,24,3), (N,24,3), (N,24,1)."""
        N = pred_s3d.shape[0]
        j3d = torch.zeros(N, 49, 3, device=pred_s3d.device)
        j3d = torch.cat([j3d[:, :25], pred_s3d], dim=1)
        kp = torch.zeros(N, 49, 3, device=pred_s3d.device)
        kp[:, 25:, 2:3] = conf
        gt = torch.cat([gt_s3d, torch.ones(N, 24, 1, device=gt_s3d.device)], dim=-1)
        w = [0.0] * 8
        w[7] = 1.0
        total, _ = losses.loss_multi(torch.zeros(N, 49, 2, device=j3d.device), j3d, torch.zeros(N, 24, 3, 3, device=j3d.device),
                                     torch.zeros(N, 10, device=j3d.device), w, kp=kp, gt_s3d=gt)
        return total

    def _frame_losses(self, pred_s2d, pred_s3d, pred_rotmat, pred_shape, gt_keypoints_2d, tag):
        o = self.options
        w = [o.s2dloss_weight, o.shape_prior_weight, o.pose_prior_weight, 0, 0, 0, 0, 0]
        total, t = losses.loss_multi(pred_s2d, pred_s3d, pred_rotmat, pred_shape, w, prior=self.gmm_f, kp=gt_keypoints_2d)
        self.fit_losses[f'{tag}/s2dloss'], self.fit_losses[f'{tag}/shape_prior'] = t[0], t[1]
        self.fit_losses[f'{tag}/pose_prior'], self.fit_losses[f'{tag}/unlabelloss'] = t[2], total
        return total, t[0]

    def cal_teacher_loss(self, image, pred_rotmat, pred_shape, pred_s2d, pred_s3d):
        with torch.no_grad():
            ema_rotmat, ema_shape, ema_cam = self.teacher(image)
            ema_s3d = self.decode_smpl_params(ema_rotmat, ema_shape)['s3d']
            ema_s2d = self.projection(ema_cam, ema_s3d)['normed']
        total, t = losses.loss_multi(pred_s2d, pred_s3d, pred_rotmat, pred_shape, [0, 0, 0, 5, 5, 0.001, 1, 0], t_p2d=ema_s2d,
                                     t_j3d=ema_s3d, t_beta=ema_shape, t_R=ema_rotmat)
        self.fit_losses.update({'teacher/s2dloss': t[3], 'teacher/s3dloss': t[4], 'teacher/shape_loss': t[5],
                                'teacher/pose_loss': t[6], 'teacher/loss': total})
        return total

    def adapt_on_labeled_data(self, model, batch, prefix='ll'):
        gt_s2d = batch['keypoints']
        pred_rotmat, pred_shape, pred_cam, label_feats = model(batch['img'], need_feature=True)
        pred_s3d = self.decode_smpl_params(pred_rotmat, pred_shape)['s3d']
        gt_rotmat = batch_rodrigues(batch['pose'].view(-1, 3)).view(-1, 24, 3, 3)
        pred_s2d = self.projection(pred_cam, pred_s3d)['normed']
        assert batch['pose_3d'].shape[1] == 24
        total, t = losses.loss_multi(pred_s2d, pred_s3d, pred_rotmat, pred_shape, [5, 0, 0, 0, 0, 0.001, 1, 5], kp=gt_s2d,
                                     t_beta=batch['betas'], t_R=gt_rotmat, gt_s3d=batch['pose_3d'])
        self.fit_losses.update({f'{prefix}/labled_s2dloss': t[0], f'{prefix}/labled_s3dloss': t[7],
                                f'{prefix}/labled_shape_loss': t[5], f'{prefix}/labled_pose_loss': t[6],
                                f'{prefix}/labled_loss': total})
        return total, label_feats

    def cal_motion_loss(self, model, pred_s2d, gt_s2d, prefix='ul', full=None):
        """reference :379-398.  ``pred_s2d`` / ``gt_s2d`` are the [25:] slices the reference passes; the kernel
        works on the full 49-joint arrays, so callers inside this class hand those over via ``full``."""
        hist_image, hist_s2d = self.get_hist()
        h_rotmat, h_shape, h_cam = model(hist_image)
        h_s3d = self.decode_smpl_params(h_rotmat, h_shape)['s3d']
        h_pred_s2d = self.projection(h_cam, h_s3d)['normed']
        if full is not None:
            cur_p, cur_kp = full
        else:   # slices were passed: pad the 25 OpenPose joints back (they carry no loss)
            pad2 = torch.zeros(pred_s2d.shape[0], 25, 2, device=pred_s2d.device)
            pad3 = torch.zeros(gt_s2d.shape[0], 25, 3, device=gt_s2d.device)
            cur_p, cur_kp = torch.cat([pad2, pred_s2d], 1), torch.cat([pad3, gt_s2d], 1)
        loss = losses.loss_motion(cur_p, h_pred_s2d, cur_kp, hist_s2d)
        self.fit_losses[f'{prefix}/motion_loss'] = loss
        return loss

    # ------------------------------------------------------------------ levels (reference :222-317)
    def _level(self, image, gt_keypoints_2d, learner, lower):
        o = self.options
        tag = 'll' if lower else 'ul'
        pred_rotmat, pred_shape, pred_cam, init_features = learner(image, need_feature=True)
        pred_s3d = self.decode_smpl_params(pred_rotmat, pred_shape)['s3d']
        pred_s2d = self.projection(pred_cam, pred_s3d)['normed']
        use_frame = o.use_frame_losses_lower if lower else o.use_frame_losses_upper
        use_temporal = o.use_temporal_losses_lower if lower else o.use_temporal_losses_upper
        loss = None
        if use_frame:
            loss, s2dloss = self._frame_losses(pred_s2d, pred_s3d, pred_rotmat, pred_shape, gt_keypoints_2d, tag)
            if lower:
                self.kp2dlosses_lower.append(s2dloss.item())
            else:
                self.kp2dlosses_upper[self.global_step] = s2dloss.item()
        if use_temporal:
            if o.use_meanteacher:
                tl = self.cal_teacher_loss(image, pred_rotmat, pred_shape, pred_s2d, pred_s3d) * o.teacherloss_weight
                loss = tl if loss is None else loss + tl
            if o.use_motion and (self.global_step - o.interval) > 0:
                ml = self.cal_motion_loss(learner, None, None, prefix='ul', full=(pred_s2d, gt_keypoints_2d))
                loss = loss + ml * o.motionloss_weight
        h36m_batch = None
        if o.retrieval:
            h36m_batch = self.retrieval(init_features[5])
        if (o.lower_level_mixtrain if lower else o.upper_level_mixtrain):
            lableloss, _ = self.adapt_on_labeled_data(learner, h36m_batch, prefix=tag)
            loss = loss + lableloss * o.labelloss_weight
        return loss, init_features

    def lower_level_adaptation(self, image, gt_keypoints_2d, h36m_batch, learner=None):
        return self._level(image, gt_keypoints_2d, learner, True)

    def upper_level_adaptation(self, image, gt_keypoints_2d, h36m_batch, learner=None):
        return self._level(image, gt_keypoints_2d, learner, False)

    def inference(self, batch, model, need_feature=False):
        pass

    def save_results(self, vts, cam_trans, images, name, bbox, prefix=None):
        """reference :429-443: draws each adapted mesh over its original frame (``imgdir/name[i]``) on the GPU and writes
        ``exppath/image/{prefix}_{global_step + i}.png``, plus the mesh as ``demo.obj`` in the working directory.  Like the
        reference, the mesh colour (205, 129, 98) / 255 is given in RGB order and drawn into the BGR frame cv2 reads, so
        the PNGs match the reference's.  ``images`` is unused (the reference un-normalises it and discards the result)."""
        import cv2
        from .render import Renderer, convert_crop_cam_to_orig_img
        cam = cam_trans.detach().cpu().numpy()
        bbox = bbox.detach().cpu().numpy() if torch.is_tensor(bbox) else np.asarray(bbox)
        for i in range(vts.shape[0]):
            oriimg = cv2.imread(os.path.join(self.imgdir, name[i]))
            if oriimg is None:
                raise FileNotFoundError(os.path.join(self.imgdir, name[i]))
            ori_h, ori_w = oriimg.shape[:2]
            ori_pred_cams = convert_crop_cam_to_orig_img(cam, bbox, ori_w, ori_h)
            frame = torch.from_numpy(oriimg).to(self.device)
            renderer = Renderer(resolution=(ori_w, ori_h), orig_img=True, wireframe=False)
            rendered = renderer.render(frame, vts[i], ori_pred_cams[i], color=np.array([205, 129, 98]) / 255, mesh_filename='demo.obj')
            cv2.imwrite(osp.join(self.exppath, 'image', f'{prefix}_{self.global_step + i}.png'), rendered.cpu().numpy())

    def write_summaries(self, losses_dict):
        for name, val in losses_dict.items():
            self.summary_writer.add_scalar(name, float(np.mean(np.asarray(val.detach().cpu() if torch.is_tensor(val) else val))),
                                           self.global_step)
