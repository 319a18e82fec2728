"""The RANSAC ground filter of the baseline preprocessing (the reference's src/utils/ransac.py, Ransac + LSLinearRegressor,
as src/dtu_3d_process.py:36-41 runs it) restated in float64 numpy, from given sample indices.

The plane z = a + b x + c y of each hypothesis is solved with the operations of csrc/dbw_ransac_math.cuh in the same order
(sums over the sample in sample order, six cofactors, adjugate / determinant), so `solve(...).astype(np.float32)` is the
kernel's float32 parameters bit for bit.  Residuals and the predicate r^2 < thresh are then taken in float64.

Which points sit on the threshold depends on rounding: the kernel rounds the parameters to float32 and evaluates in float32;
the reference inverts X^T X in float32, which adds float32 rounding times the conditioning of X^T X.  `boundary` lists, per
hypothesis, the points whose squared residual lies within such rounding of the threshold; a count computed either way may
differ from the float64 count on exactly those points."""
import numpy as np

U32 = 2.0 ** -24            # float32 unit roundoff


def solve(points, idx):
    """(H, 3) float64 (a, b, c) and (H,) float64 determinant of X^T X for the hypotheses idx (H, P) into points (N, 3) float32;
    NaN parameters where the determinant is exactly 0"""
    p = np.asarray(points, np.float32).astype(np.float64)[np.asarray(idx, np.int64)]          # (H, P, 3)
    H = p.shape[0]
    s1 = sx = sy = sxx = sxy = syy = sz = sxz = syz = np.zeros(H)
    for k in range(p.shape[1]):
        x, y, z = p[:, k, 0], p[:, k, 1], p[:, k, 2]
        s1, sx, sy = s1 + 1.0, sx + x, sy + y
        sxx, sxy, syy = sxx + x * x, sxy + x * y, syy + y * y
        sz, sxz, syz = sz + z, sxz + x * z, syz + y * z
    c00, c01, c02 = sxx * syy - sxy * sxy, sxy * sy - sx * syy, sx * sxy - sxx * sy
    c11, c12, c22 = s1 * syy - sy * sy, sx * sy - s1 * sxy, s1 * sxx - sx * sx
    det = (s1 * c00 + sx * c01) + sy * c02
    with np.errstate(divide='ignore', invalid='ignore'):
        a = ((c00 * sz + c01 * sxz) + c02 * syz) / det
        b = ((c01 * sz + c11 * sxz) + c12 * syz) / det
        c = ((c02 * sz + c12 * sxz) + c22 * syz) / det
    params = np.stack([a, b, c], 1)
    params[det == 0] = np.nan
    return params, det


def condition(points, idx):
    """(H,) 2-norm condition number of each hypothesis's X^T X (inf when singular)"""
    p = np.asarray(points, np.float32).astype(np.float64)[np.asarray(idx, np.int64)]
    X = np.concatenate([np.ones_like(p[..., :1]), p[..., :2]], -1)
    with np.errstate(divide='ignore', invalid='ignore'):
        return np.linalg.cond(np.einsum('hpi,hpj->hij', X, X))


def residuals(points, abc):
    """(N,) float64 z - ((a + b x) + c y) of one hypothesis"""
    p = np.asarray(points, np.float32).astype(np.float64)
    a, b, c = (float(v) for v in abc)
    with np.errstate(invalid='ignore', over='ignore'):
        return p[:, 2] - ((a + b * p[:, 0]) + c * p[:, 1])


def inliers(points, abc, thresh):
    with np.errstate(invalid='ignore', over='ignore'):
        return residuals(points, abc) ** 2 < thresh


def boundary(points, abc, thresh, kappa=1.0):
    """indices of the points whose squared residual lies within float32 rounding of `thresh`: parameters known to
    8 u kappa relative (kappa = 1 for a float64 solve rounded to float32, the condition number of X^T X for a float32 solve),
    and every operation of the residual rounded to float32.  Every point of a hypothesis with non-finite parameters or
    condition counts as boundary."""
    p = np.asarray(points, np.float32).astype(np.float64)
    a, b, c = (float(v) for v in abc)
    if not (np.isfinite([a, b, c]).all() and np.isfinite(kappa)):
        return np.arange(len(p))
    with np.errstate(invalid='ignore', over='ignore'):
        m = kappa * ((abs(a) + np.abs(b * p[:, 0])) + np.abs(c * p[:, 1])) + np.abs(p[:, 2])
        band = 2 * np.sqrt(thresh) * 8 * U32 * m + 4 * U32 * thresh
        return np.nonzero(np.abs(residuals(p, (a, b, c)) ** 2 - thresh) <= band)[0]


def counts(points, params, thresh):
    """(H,) int64 float64 inlier counts"""
    return np.array([int(inliers(points, abc, thresh).sum()) for abc in params], np.int64)


def select(counts, batch_size):
    """Ransac.fit's choice: (index of best_models[-1] or -1, its count, len(best_models))"""
    best, best_n, improvements = -1, 0, 0
    counts = np.asarray(counts)
    for r0 in range(0, len(counts) - batch_size + 1, batch_size):
        arg = r0 + int(np.argmax(counts[r0:r0 + batch_size]))          # first maximum
        if counts[arg] > best_n:
            best, best_n, improvements = arg, int(counts[arg]), improvements + 1
    return best, best_n, improvements


def ransac(points, idx, batch_size=10, thresh=1e-3):
    """the whole filter in float64 from the sample indices idx (H, P): parameters, counts, the choice and the kept cloud"""
    params, det = solve(points, idx)
    n = counts(points, params, thresh)
    best, best_n, improvements = select(n, batch_size)
    keep = ~inliers(points, params[best], thresh) if best >= 0 else np.ones(len(points), bool)
    return dict(params=params, det=det, counts=n, best=best, best_n=best_n, improvements=improvements, keep=keep,
                kept=np.asarray(points, np.float32)[keep])
