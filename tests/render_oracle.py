"""numpy restatements of the point viewer's host steps (utils/show3d_balls.py showpoints), one cloud and one view at a
time, in showpoints' own operations: the view transform (:27-29, :52-74) and magnifyBlue (:88-94)."""
import numpy as np


def project_np(xyz, size=800, xangle=0.0, yangle=0.0, zoom=1.0):
    """(n, 3) float64 before the int32 truncation, and the truncated (n, 3) int32."""
    xyz = np.asarray(xyz, np.float64)
    xyz = xyz - xyz.mean(axis=0)
    radius = ((xyz ** 2).sum(axis=-1) ** 0.5).max()
    xyz = xyz / ((radius * 2.2) / size)
    rotmat = np.eye(3)
    rotmat = rotmat.dot(np.array([[1.0, 0.0, 0.0],
                                  [0.0, np.cos(xangle), -np.sin(xangle)],
                                  [0.0, np.sin(xangle), np.cos(xangle)]]))
    rotmat = rotmat.dot(np.array([[np.cos(yangle), 0.0, -np.sin(yangle)],
                                  [0.0, 1.0, 0.0],
                                  [np.sin(yangle), 0.0, np.cos(yangle)]]))
    rotmat = rotmat * zoom
    nxyz = xyz.dot(rotmat) + [size / 2, size / 2, 0]
    return nxyz, nxyz.astype("int32")


def magnify_np(show, level):
    show = show.copy()
    if level > 0:
        show[:, :, 0] = np.maximum(show[:, :, 0], np.roll(show[:, :, 0], 1, axis=0))
        if level >= 2:
            show[:, :, 0] = np.maximum(show[:, :, 0], np.roll(show[:, :, 0], -1, axis=0))
        show[:, :, 0] = np.maximum(show[:, :, 0], np.roll(show[:, :, 0], 1, axis=1))
        if level >= 2:
            show[:, :, 0] = np.maximum(show[:, :, 0], np.roll(show[:, :, 0], -1, axis=1))
    return show


def normalize_np(colors):
    """showpoints' normalizecolor on float64 colour rows (part_seg/test.py's colour-map rows), rounded to float32."""
    c = np.asarray(colors, np.float64).copy()
    for k in range(3):
        c[:, k] /= (c[:, k].max() + 1e-14) / 255.0
    return c.astype(np.float32)


def near_integer_mismatches(nxyz, got, want, tol=1e-9):
    """(allowed, unexplained) counts of coordinates where got != want: allowed when the float64 value lies within
    ``tol`` of an integer (a last-bit difference in the rotation can move it across)."""
    diff = got != want
    near = np.abs(nxyz - np.round(nxyz)) <= tol
    return int((diff & near).sum()), int((diff & ~near).sum())
