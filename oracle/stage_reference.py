"""Stage the reference's unmodified files into the git-ignored ``oracle/_ref/`` (called by ``__graft_entry__.build()``).

The unchanged-driver tests (tests/test_gpu_dropin_driver.py, tests/test_gpu_internet.py) execute the reference's own
``dynaboa_benchmark.py`` / ``dynaboa_internet.py`` on the drop-in tree, and the CPU arm of ``bench.py`` times the reference's
own code (oracle/ref_harness.py).  Those files are not part of this repository; they are read from a reference checkout
(DBOA_REFERENCE_ROOT, default /root/reference) at build time and copied with a sha256 manifest.  Without a checkout nothing is
staged, the two tests skip and the CPU arm times the oracle port.
"""
import hashlib
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, '_ref')
FILES = ['dynaboa_benchmark.py', 'dynaboa_internet.py', 'base_adaptor.py', 'constants.py', 'config.py', 'model/__init__.py', 'model/hmr.py',
         'model/smpl.py', 'utils/__init__.py', 'utils/geometry.py', 'utils/pose_utils.py', 'utils/dataprocess.py', 'utils/smplify/__init__.py',
         'utils/smplify/prior.py', 'utils/smplify/smplify.py', 'utils/smplify/losses.py', 'boa_dataset/__init__.py', 'boa_dataset/pw3d.py',
         'boa_dataset/internet_data.py', 'data/gmm_08.pkl']


def source_root():
    root = os.environ.get('DBOA_REFERENCE_ROOT') or '/root/reference'
    try:
        return root if os.path.isfile(os.path.join(root, 'dynaboa_benchmark.py')) else None
    except OSError:
        return None


def stage():
    """Copy FILES from the reference checkout into oracle/_ref/; returns the destination, or None without a checkout."""
    src_root = source_root()
    if src_root is None:
        return None
    manifest = []
    for rel in FILES:
        src, dst = os.path.join(src_root, rel), os.path.join(DST, rel)
        if not os.path.isfile(src):
            continue
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        with open(src, 'rb') as f:
            manifest.append(f'{hashlib.sha256(f.read()).hexdigest()}  {rel}')
    with open(os.path.join(DST, 'MANIFEST.sha256'), 'w') as f:
        f.write('\n'.join(manifest) + '\n')
    return DST


if __name__ == '__main__':
    print(stage() or 'no reference checkout: nothing staged')
