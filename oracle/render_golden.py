"""Golden vectors of the mesh overlay's camera conversion (run where a reference checkout is available; DBOA_REFERENCE_ROOT
names it).

    python -m oracle.render_golden          # writes tests/golden/render_cam.npz

render_demo.py cannot be imported (it loads pyrender / trimesh / EGL at import time), so ``convert_crop_cam_to_orig_img`` and
``parse_cam`` are taken out of its syntax tree and exactly those two functions are executed on seeded inputs.  They are the
only part of rendering the reference's own code can pin; the rasteriser itself is restated in oracle/render_ref.py.
The reference is read at run time and never copied.  Test infrastructure only.
"""
import ast
import os

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get('DBOA_REFERENCE_ROOT', '')
OUT = os.path.join(REPO, 'tests', 'golden')


def load_render_functions(ref=REF):
    path = os.path.join(ref, 'render_demo.py')
    tree = ast.parse(open(path).read())
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ('convert_crop_cam_to_orig_img', 'parse_cam')]
    ns = {'np': np}
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, 'exec'), ns)
    return ns['convert_crop_cam_to_orig_img'], ns['parse_cam']


def golden_render_cam():
    convert, parse_cam = load_render_functions()
    rng = np.random.default_rng(2024)
    B = 16
    cam = np.stack([rng.uniform(0.5, 1.3, B), rng.uniform(-0.3, 0.3, B), rng.uniform(-0.3, 0.3, B)], 1)
    bbox = np.stack([rng.uniform(50, 1800, B), rng.uniform(50, 1000, B), rng.uniform(80, 900, B)], 1)
    sizes = np.array([[1920, 1080], [320, 240], [640, 480]])
    orig = np.stack([convert(cam, bbox, int(w), int(h)) for w, h in sizes])
    np.savez_compressed(os.path.join(OUT, 'render_cam.npz'), cam=cam, bbox=bbox, sizes=sizes, orig_cam=orig, parse_cam=parse_cam(cam))
    print('render_cam.npz ok')


if __name__ == '__main__':
    golden_render_cam()
