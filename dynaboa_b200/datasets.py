"""Frame sources with the dict keys of the reference datasets (boa_dataset/pw3d.py:115-125,
boa_dataset/internet_data.py).

There are no licensed datasets on the build or GPU boxes, so these classes serve the seeded synthetic stream of
``dynaboa_b200.synthetic`` -- and ONLY when the caller opts in: the unchanged reference driver run with ``--dataset 3dpw``
would otherwise report MPJPE / PA-MPJPE / PVE on synthetic frames without saying so.  Opt in with
``options.synthetic_frames = N`` (tests, bench) or ``DBOA_SYNTHETIC_FRAMES=N`` in the environment (unchanged driver).
Real crops go through ``dynaboa_b200.dataprocess`` (GPU crop / resize / normalise, the step before the hot path).

``internet_videos(root)`` reads the same folder as one ``InternetVideo`` per sequence instead of one concatenated stream: the
input of a pool that adapts the sequences side by side (``internet.MultiInternetAdaptor``)."""
import os
import warnings

from torch.utils.data import Dataset

from . import synthetic


def _synthetic_frames(options):
    n = getattr(options, 'synthetic_frames', None) if options is not None else None
    if n is None and os.environ.get('DBOA_SYNTHETIC_FRAMES'):
        n = int(os.environ['DBOA_SYNTHETIC_FRAMES'])
    if n is None:
        raise RuntimeError('no dataset files are configured and the synthetic stand-in stream was not requested: set '
                           'options.synthetic_frames (or DBOA_SYNTHETIC_FRAMES=N) to run on the seeded SYNTHETIC stream; metrics '
                           'computed on it are not 3DPW numbers')
    return int(n)


class PW3D(Dataset):
    def __init__(self, options=None):
        n = _synthetic_frames(options)
        warnings.warn(f'dynaboa_b200.datasets.PW3D: serving {n} SYNTHETIC frames (seeded stand-in for 3DPW); '
                      'the reported metrics are not 3DPW results', stacklevel=2)
        seed = getattr(options, 'seq_seed', synthetic.SEED) if options is not None else synthetic.SEED
        rank = getattr(options, 'rank', 0) if options is not None else 0
        self.stream = synthetic.SyntheticStream(length=n, batch_size=1, seed=seed, rank=rank)

    def __len__(self):
        return len(self.stream)

    def __getitem__(self, i):
        f = self.stream[i]
        item = {}
        for k, v in f.items():
            item[k] = v[0]
        return item


class Internet_dataset(Dataset):
    """Frames of an Internet video (reference boa_dataset/internet_data.py:16-88): ``<root>/*.npz`` with ``imgname``, ``center``,
    ``scale``, ``part`` (49 x 3 pixel keypoints) and the images under ``<root>/images``.  Decoding stays on the host (cv2); the
    crop / resize / normalise and the keypoint transform run on the GPU (``dynaboa_b200.dataprocess``), so an item is already
    device resident.  Without such files the seeded synthetic stream is served -- only on explicit request, like ``PW3D``."""

    def __init__(self, options=None):
        import glob
        import os.path as osp

        import numpy as np

        from . import config
        root = os.environ.get('DYNABOA_INTERNET_ROOT', config.InternetData_ROOT)
        names = sorted(glob.glob(osp.join(root, '*.npz')))
        self.real = len(names) > 0
        if not self.real:
            n = _synthetic_frames(options)
            warnings.warn(f'dynaboa_b200.datasets.Internet_dataset: no *.npz under {root}; serving {n} SYNTHETIC frames', stacklevel=2)
            self.stream = synthetic.SyntheticStream(length=n, batch_size=1, seed=getattr(options, 'seq_seed', synthetic.SEED))
            return
        self.imgdir = osp.join(root, 'images')
        data = [np.load(f) for f in names]
        self.imgnames = np.concatenate([d['imgname'] for d in data], 0)
        self.scales = np.concatenate([d['scale'] for d in data], 0)
        self.centers = np.concatenate([d['center'] for d in data], 0)
        self.smpl_j2ds = np.concatenate([d['part'] for d in data], 0)

    def __len__(self):
        return len(self.stream) if not self.real else int(self.scales.shape[0])

    def __getitem__(self, i):
        if not self.real:
            return {k: v[0] for k, v in self.stream[i].items()}
        import cv2
        import numpy as np
        import torch

        from . import dataprocess
        name = str(self.imgnames[i])
        bgr = cv2.imread(os.path.join(self.imgdir, name))
        if bgr is None:
            raise FileNotFoundError(os.path.join(self.imgdir, name))
        rgb = torch.from_numpy(np.ascontiguousarray(bgr[:, :, ::-1])).cuda()             # uint8 (H, W, 3): 1 byte per value over PCIe
        center, scale = [float(self.centers[i][0]), float(self.centers[i][1])], float(self.scales[i])
        kp = torch.from_numpy(np.asarray(self.smpl_j2ds[i], dtype=np.float32)).cuda()
        return {'image': dataprocess.crop(rgb, center, scale), 'imgname': name, 'smpl_j2d': dataprocess.j2d_processing(kp, center, scale),
                'bbox': np.stack([center[0], center[1], scale * 200])}


INTERNET_KEYS = ('imgname', 'center', 'scale', 'part')


class InternetVideo:
    """One Internet sequence on the host: ``name`` (its npz's file name without ``.npz``), the per-frame records of the npz
    (``imgnames``, ``centers`` (n, 2), ``scales`` (n,), ``parts`` (n, 49, 3) pixel keypoints) and the directory ``imgdir`` of
    its frames.  No frame is decoded here.  ``frame(t)`` gives frame t's record: the path, and the box and keypoints as
    ``Internet_dataset.__getitem__`` reads them."""

    def __init__(self, path, imgdir):
        import os.path as osp

        import numpy as np
        self.path, self.imgdir = path, imgdir
        self.name = osp.splitext(osp.basename(path))[0]
        try:
            with np.load(path) as d:
                arrays = {k: np.asarray(d[k]) for k in INTERNET_KEYS if k in d.files}
        except Exception as e:                              # not a zip, a pickled object, a truncated file
            raise ValueError(f'{path}: not a readable npz ({type(e).__name__}: {e})') from e
        missing = [k for k in INTERNET_KEYS if k not in arrays]
        if missing:
            raise ValueError(f'{path}: missing {", ".join(missing)} (expected {", ".join(INTERNET_KEYS)})')
        self.imgnames, self.centers, self.scales, self.parts = (arrays[k] for k in INTERNET_KEYS)
        if self.imgnames.ndim != 1:
            raise ValueError(f'{path}: imgname of shape {tuple(self.imgnames.shape)}, expected one name per frame')
        n = len(self.imgnames)
        for k, v, shape in (('center', self.centers, (n, 2)), ('scale', self.scales, (n,)), ('part', self.parts, (n, 49, 3))):
            if tuple(v.shape) != shape:
                raise ValueError(f'{path}: {k} of shape {tuple(v.shape)}, expected {shape} for {n} frames')

    def __len__(self):
        return len(self.imgnames)

    def frame(self, t):
        """Frame t: (path, center [cx, cy], scale, (49, 3) float32 keypoints, (1, 3) float64 bbox), with the floats of
        ``Internet_dataset.__getitem__``."""
        import numpy as np
        if not 0 <= t < len(self):
            raise IndexError(f'{self.name}: frame {t} of {len(self)}')
        center, scale = [float(self.centers[t][0]), float(self.centers[t][1])], float(self.scales[t])
        return (os.path.join(self.imgdir, str(self.imgnames[t])), center, scale, np.asarray(self.parts[t], dtype=np.float32),
                np.stack([center[0], center[1], scale * 200])[None])


def internet_videos(root):
    """One ``InternetVideo`` per ``root/*.npz`` (the layout ``Internet_dataset`` reads: the reference's npz, the frames under
    ``root/images``), sorted by file name, so the videos come in ``Internet_dataset``'s order.  Raises FileNotFoundError when
    ``root`` holds no npz and ValueError for a malformed one."""
    import glob
    import os.path as osp
    if not osp.isdir(root):
        raise FileNotFoundError(f'{root} is not a directory')
    names = sorted(glob.glob(osp.join(root, '*.npz')))
    if not names:
        raise FileNotFoundError(f'no *.npz sequence under {root}')
    return [InternetVideo(p, osp.join(root, 'images')) for p in names]
