"""oracle/make_golden_arf.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_arf/.

Runs the reference's UNMODIFIED ARF class (FourierGrid/arf.py:9-89) on the CPU over seeded style images and content sets
(oracle.arf_ref) and records:

* ``style_<kind>.pt``: the 8-bit source image ('portrait' 120 x 75, 'landscape' 90 x 131), the content HW the stylizer was
  built for and the reference's ``np_style_img`` after ``load_style_img`` (two INTER_AREA resizes);
* ``set_<name>.pt``: the content set, the style it was matched to, and the reference's recoloured set and color_tf.

The reference reads its style image with ``imageio.imread`` and writes ``style_image.png`` with ``imageio.imwrite``.  imageio
is not a dependency here, so both are stubbed with cv2 (cv2.imread + BGR -> RGB, and the reverse for the write), and the style
images are stored as lossless PNG bytes.  The fixtures therefore pin the resize and the colour arithmetic, not a JPEG decoder:
whether imageio and cv2 decode one JPEG to the same pixels is not checked.

    python -m oracle.make_golden_arf      # from the repo root, where the reference checkout exists
"""
import os
import sys
import tempfile
import types

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, 'tests', 'golden', 'l2_arf')
REF = '/root/reference'
sys.path.insert(0, ROOT)

from oracle import arf_ref  # noqa: E402

SEED = 777
HW = (48, 64)                 # content frame size the stylizers are built for (long side 64)

SETS = {
    # name: (content kind, set shape, style, seed offset)
    'random': ('random', (3, 20, 28, 3), 'portrait', 0),
    'random_landscape': ('random', (2, 17, 23, 3), 'landscape', 1),
    'near_grey': ('near_grey', (3, 20, 28, 3), 'landscape', 2),
    'constant': ('constant', (2, 16, 16, 3), 'portrait', 3),
    'one_pixel': ('random', (1, 1, 1, 3), 'landscape', 4),
    'outside': ('outside', (2, 19, 21, 3), 'portrait', 5),
}


def imread_rgb(path):
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    return np.ascontiguousarray(img[..., ::-1])


def write_png_bytes(path, rgb):
    """Lossless PNG bytes under any file name (cv2.imread goes by the content, not the extension)."""
    ok, buf = cv2.imencode('.png', np.ascontiguousarray(rgb[..., ::-1]))
    assert ok
    buf.tofile(path)


def _reference_arf():
    sys.modules['imageio'] = types.SimpleNamespace(imread=imread_rgb,
                                                   imwrite=lambda p, a: cv2.imwrite(p, np.ascontiguousarray(a[..., ::-1])))
    sys.path.insert(0, REF)
    from FourierGrid import arf
    return arf.ARF


class Cfg(dict):
    def __getattr__(self, k):
        return self[k]


def _save(name, obj):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name)
    torch.save(obj, path)
    print(f'{name}: {os.path.getsize(path) / 1024:.1f} KiB')


def main():
    ARF = _reference_arf()
    data_dict = {'HW': np.array([HW] * 2)}
    with tempfile.TemporaryDirectory() as tmp:
        stylizers = {}
        for i, kind in enumerate(('portrait', 'landscape')):
            src = arf_ref.style_source(kind, SEED + i)
            root = os.path.join(tmp, kind)
            os.makedirs(root)
            write_png_bytes(os.path.join(root, '34.jpg'), src)
            st = ARF(Cfg(arf=Cfg(style_root=root, style_id=34)), data_dict, 'cpu')
            stylizers[kind] = st
            _save(f'style_{kind}.pt', dict(source=src, HW=HW, np_style_img=st.np_style_img))
        for name, (kind, shape, style, off) in SETS.items():
            x = arf_ref.content_set(kind, shape, SEED + 10 + off)
            out, tf = stylizers[style].match_colors_for_image_set(x.copy(), tmp)
            _save(f'set_{name}.pt', dict(kind=kind, style=style, image_set=x, out=out.numpy(), color_tf=tf.numpy()))


if __name__ == '__main__':
    main()
