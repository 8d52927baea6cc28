"""The colour-transfer stylizer of the render step (FourierGrid/arf.py, from Artistic Radiance Fields).

``ARF`` has the reference's constructor, attributes and ``match_colors_for_image_set`` with the reference's result types.  The
set's and the style image's moments come from ``ubn_color_moments`` (fp64 sums about the first pixel, fixed reduction order) and
the transform is applied by ``ubn_color_affine`` (csrc/color.cu): one read of the set for the moments, one read and one write for
the transform, and no set-sized temporary beyond the upload of a numpy set.  The two 3 x 3 SVDs between them run on the host in
fp64, and T, b are rounded to fp32 once.

Differences from the reference, each deliberate:

* the style image is read with cv2 (BGR -> RGB, then / 255 in float32) instead of imageio, which is not a dependency here; a
  file that is missing raises FileNotFoundError and anything but an 8-bit, 3-channel image ValueError;
* the covariances are fp64 (the reference's are one fp32 matmul over every pixel, whose error 1 / sqrt(sigma) amplifies where the
  set is nearly grey), so the transform is the fp64 one rounded to fp32;
* an empty set or style image, and a set or style image whose moments are not finite (a NaN or inf pixel), raise ValueError
  naming which one; the reference divides by zero or hands NaN to the SVD;
* only float32 numpy arrays and float32 CUDA tensors are accepted (TypeError otherwise), and the device must be a CUDA device:
  there is no CPU path."""
import ctypes
import os

import cv2
import numpy as np
import torch

from . import _cabi
from .ops import _Guard

SIG_MIN, SIG_MAX = 1e-8, 1e8          # arf.py:77-78


def _packed(t):
    if t.dtype != torch.float32 or not t.is_cuda or t.shape[-1] != 3:
        raise TypeError(f'expected a float32 CUDA tensor of shape [..., 3], got {t.dtype} on {t.device} of shape '
                        f'{tuple(t.shape)}')
    return t if t.is_contiguous() else t.contiguous()


def color_moments(pixels):
    """(mean [3], covariance [3, 3]) as float64 numpy arrays of the packed RGB pixels of a float32 CUDA tensor [..., 3] with at
    least one pixel: the population moments of arf.py:65-69, accumulated in fp64 by ubn_color_moments on the caller's stream."""
    t = _packed(pixels)
    n = t.numel() // 3
    if n == 0:
        raise ValueError('no pixels')
    scratch = torch.empty(9 * _cabi.COLOR_MAX_CTAS, dtype=torch.float64, device=t.device)
    out = torch.empty(9, dtype=torch.float64, device=t.device)
    with _Guard(t) as lib:
        _cabi.check(lib.ubn_color_moments(_cabi.ptr(t), _cabi.c_i64(n), _cabi.ptr(scratch), _cabi.ptr(out), _cabi.stream_of(t)))
    m = out.cpu().numpy()
    c00, c01, c02, c11, c12, c22 = m[3:]
    return m[:3].copy(), np.array([[c00, c01, c02], [c01, c11, c12], [c02, c12, c22]])


def color_affine(pixels, T, b, out=None):
    """clamp(T x + b, 0, 1) of every packed RGB pixel of a float32 CUDA tensor [..., 3] (ubn_color_affine), into ``out`` (same
    shape, contiguous; may be ``pixels`` itself) or a new tensor.  T [3, 3] and b [3] are rounded to float32."""
    t = _packed(pixels)
    if out is None:
        out = torch.empty_like(t, memory_format=torch.contiguous_format)
    elif out.dtype != torch.float32 or out.device != t.device or out.shape != t.shape or not out.is_contiguous():
        raise ValueError('out must be a contiguous float32 tensor of the input\'s shape on its device')
    Tf = (ctypes.c_float * 9)(*np.asarray(T, np.float32).reshape(9).tolist())
    bf = (ctypes.c_float * 3)(*np.asarray(b, np.float32).reshape(3).tolist())
    with _Guard(t) as lib:
        _cabi.check(lib.ubn_color_affine(_cabi.ptr(t), _cabi.ptr(out), _cabi.c_i64(t.numel() // 3), Tf, bf, _cabi.stream_of(t)))
    return out


def color_transform(mu_c, cov_c, mu_s, cov_s):
    """(T, b) in float64 of arf.py:71-81: T = U_s diag(sqrt(sig_s)) U_s^T U_c diag(1 / sqrt(sig_c)) U_c^T with the singular values
    clamped to [1e-8, 1e8], b = mu_s - T mu_c.  U f(Sigma) U^T does not depend on the sign or the basis an SVD picks within an
    eigenspace, so numpy's SVD gives the reference's transform."""
    u_c, sig_c, _ = np.linalg.svd(cov_c)
    u_s, sig_s, _ = np.linalg.svd(cov_s)
    scl_c = 1.0 / np.sqrt(np.clip(sig_c, SIG_MIN, SIG_MAX))
    scl_s = np.sqrt(np.clip(sig_s, SIG_MIN, SIG_MAX))
    T = (u_s * scl_s) @ u_s.T @ (u_c * scl_c) @ u_c.T
    return T, mu_s - T @ mu_c


def _checked_moments(pixels, what):
    if pixels.numel() == 0:
        raise ValueError(f'the {what} is empty')
    mu, cov = color_moments(pixels)
    if not (np.isfinite(mu).all() and np.isfinite(cov).all()):
        raise ValueError(f'the {what} has non-finite moments (a NaN or inf pixel): mean {mu}, covariance {cov.tolist()}')
    return mu, cov


class ARF:
    """FourierGrid/arf.py:9-89 on the GPU; see the module docstring."""

    def __init__(self, cfg, data_dict, device):
        assert 'arf' in cfg, "ARF should not be initialized according to cfg!"
        self.style_root = cfg.arf.style_root
        self.style_id = cfg.arf.style_id
        style_img_p = os.path.join(self.style_root, str(self.style_id) + ".jpg")
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise ValueError(f'ARF runs on a CUDA device only, got {self.device}')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        # assume the images are of the same height / width.
        self.w, self.h = data_dict['HW'][0][1], data_dict['HW'][0][0]
        self.np_style_img = None
        self.style_img = self.load_style_img(style_img_p)

    @staticmethod
    def read_style_image(path):
        """The 8-bit RGB image at ``path`` as float32 in [0, 1] (imageio.imread(path).astype(np.float32) / 255.0 of arf.py:27)."""
        if not os.path.isfile(path):
            raise FileNotFoundError(path)
        img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        if img is None:
            raise ValueError(f'{path}: not an image cv2 can read')
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError(f'{path}: expected an 8-bit, 3-channel image, got {img.dtype} of shape {img.shape}')
        return np.ascontiguousarray(img[..., ::-1]).astype(np.float32) / 255.0

    def load_style_img(self, style_img_p):
        # resize style image such that its long side matches the long side of content images (arf.py:25-49)
        style_img = self.read_style_image(style_img_p)
        style_h, style_w = style_img.shape[:2]
        content_long_side = max([self.w, self.h])
        if style_h > style_w:
            style_img = cv2.resize(style_img, (int(content_long_side / style_h * style_w), content_long_side),
                                   interpolation=cv2.INTER_AREA)
        else:
            style_img = cv2.resize(style_img, (content_long_side, int(content_long_side / style_w * style_h)),
                                   interpolation=cv2.INTER_AREA)
        style_img = cv2.resize(style_img, (style_img.shape[1] // 2, style_img.shape[0] // 2), interpolation=cv2.INTER_AREA)
        self.np_style_img = style_img
        return torch.from_numpy(style_img).to(device=self.device)

    def match_colors_for_image_set(self, image_set, train_save_dir):
        """arf.py:51-89.  ``image_set``: a float32 numpy array (what render_viewpoints returns) or a float32 CUDA tensor of any
        shape [..., 3].  Writes ``style_image.png`` into ``train_save_dir`` and returns (the recoloured set, a float32 CUDA tensor
        of the input's shape on self.device; color_tf, float32 [4, 4] on self.device: T in [:3, :3], b in [:3, 3]).  numpy input
        is uploaded once and recoloured in place on the device; a CUDA tensor is left untouched and the result is a new tensor.
        Kernels run on the device's current stream."""
        if isinstance(image_set, np.ndarray):
            if image_set.dtype != np.float32:
                raise TypeError(f'match_colors_for_image_set takes float32 input, got a numpy array of {image_set.dtype}')
        elif isinstance(image_set, torch.Tensor):
            if image_set.dtype != torch.float32 or not image_set.is_cuda:
                raise TypeError(f'match_colors_for_image_set takes a float32 CUDA tensor, got {image_set.dtype} on '
                                f'{image_set.device}')
        else:
            raise TypeError('match_colors_for_image_set takes a float32 numpy array or CUDA tensor, got '
                            f'{type(image_set).__name__}')
        if image_set.ndim < 1 or image_set.shape[-1] != 3:
            raise ValueError(f'expected a set of RGB pixels [..., 3], got shape {tuple(image_set.shape)}')
        if int(np.prod(image_set.shape)) == 0:
            raise ValueError('the content set is empty')
        cv2.imwrite(os.path.join(train_save_dir, "style_image.png"),
                    np.ascontiguousarray(np.clip(self.np_style_img * 255.0, 0.0, 255.0).astype(np.uint8)[..., ::-1]))
        sh = tuple(image_set.shape)
        with torch.cuda.device(self.device):
            if isinstance(image_set, np.ndarray):
                x = torch.from_numpy(np.ascontiguousarray(image_set)).to(self.device)
                out = x
            elif image_set.device == self.device:
                x = image_set
                out = None
            else:
                x = image_set.to(self.device).contiguous()
                out = x
            mu_c, cov_c = _checked_moments(x, 'content set')
            mu_s, cov_s = _checked_moments(self.style_img, 'style image')
            T, b = color_transform(mu_c, cov_c, mu_s, cov_s)
            T32, b32 = T.astype(np.float32), b.astype(np.float32)
            res = color_affine(x, T32, b32, out=out)
            color_tf = np.eye(4, dtype=np.float32)
            color_tf[:3, :3] = T32
            color_tf[:3, 3] = b32
            return res.view(sh), torch.from_numpy(color_tf).to(self.device)
