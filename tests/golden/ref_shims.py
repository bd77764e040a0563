"""Import shims that let the UNMODIFIED reference (a liuyuan-pal/Gen6D checkout, located by the
GEN6D_REFERENCE environment variable) run on a CPU-only machine.  Used by the golden-vector
generators under tests/golden/; no test imports it.  See SURVEY.md section 8(c) for why each shim exists.
"""
import sys
import types

import numpy as np

import os

REFERENCE_ROOT = os.environ.get('GEN6D_REFERENCE', '')


def _euler_axis_rotation(axis, ang):
    c, s = np.cos(ang), np.sin(ang)
    if axis == 'x':
        return np.array([[1, 0, 0], [0, c, -s], [0, s, c]], dtype=np.float64)
    if axis == 'y':
        return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=np.float64)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=np.float64)


def euler2mat(ai, aj, ak, axes='sxyz'):
    """transforms3d.euler.euler2mat for static ('s') axis triples: R = R_k @ R_j @ R_i."""
    assert axes[0] == 's'
    Ri = _euler_axis_rotation(axes[1], ai)
    Rj = _euler_axis_rotation(axes[2], aj)
    Rk = _euler_axis_rotation(axes[3], ak)
    return Rk @ Rj @ Ri


def mat2euler(mat, axes='sxyz'):
    """Only the 'szyx' decomposition is used on the path (utils/pose_utils.py:98):
    R = Rx(ak) @ Ry(aj) @ Rz(ai); returns (ai, aj, ak)."""
    assert axes == 'szyx'
    from scipy.spatial.transform import Rotation
    # static z, then y, then x  == scipy extrinsic 'zyx'
    ai, aj, ak = Rotation.from_matrix(np.asarray(mat, np.float64)).as_euler('zyx')
    return ai, aj, ak


def quat2mat(q):
    w, x, y, z = [float(v) for v in q]
    n = w * w + x * x + y * y + z * z
    if n < np.finfo(np.float64).eps:
        return np.eye(3)
    s = 2.0 / n
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ = w * X, w * Y, w * Z
    xX, xY, xZ = x * X, x * Y, x * Z
    yY, yZ, zZ = y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY],
                     [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                     [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def mat2axangle(mat):
    from scipy.spatial.transform import Rotation
    rv = Rotation.from_matrix(np.asarray(mat, np.float64)).as_rotvec()
    ang = np.linalg.norm(rv)
    axis = rv / ang if ang > 0 else np.array([1.0, 0, 0])
    return axis, ang


def mat2quat(mat):
    from scipy.spatial.transform import Rotation
    x, y, z, w = Rotation.from_matrix(np.asarray(mat, np.float64)).as_quat()
    return np.array([w, x, y, z])


def install(networks=True):
    """Put stub modules in sys.modules, neutralise .cuda(), patch the VGG download.
    networks=False: only the stubs for the absent third-party packages (the reference's own `network`
    package is not imported and torch is left untouched), for a caller that puts gen6d_b200.network in
    its place."""
    if not os.path.isfile(os.path.join(REFERENCE_ROOT, 'estimator.py')) or not os.path.isdir(os.path.join(REFERENCE_ROOT, 'network')):
        raise RuntimeError(f'GEN6D_REFERENCE={REFERENCE_ROOT!r} is not a liuyuan-pal/Gen6D checkout')
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)

    def mod(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    mod('plyfile', PlyData=object)
    sk = mod('skimage')
    sk.io = mod('skimage.io', imread=None, imsave=None)
    t3 = mod('transforms3d')
    t3.euler = mod('transforms3d.euler', euler2mat=euler2mat, mat2euler=mat2euler)
    t3.quaternions = mod('transforms3d.quaternions', quat2mat=quat2mat, mat2quat=mat2quat)
    t3.axangles = mod('transforms3d.axangles', mat2axangle=mat2axangle)

    if not networks:
        return
    import torch
    import torchvision
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self

    import network.pretrain_models as pm  # noqa: E402  (reference module)
    if not getattr(pm.models.vgg11_bn, '_g6d_offline', False):
        _orig = torchvision.models.vgg11_bn

        def _vgg11_bn_offline(*a, **k):
            return _orig(weights=None)
        _vgg11_bn_offline._g6d_offline = True
        pm.models.vgg11_bn = _vgg11_bn_offline
