"""numpy float64 restatement of the Gaussian-splat export (include/ngp_b200.h, "Gaussian-splat export"; csrc/splats.cu):
the Fibonacci direction set, 3DGS's real SH basis, the weighted ridge fit, the splat geometry and opacity, and a
per-pixel brute-force version of the forward rasteriser under the same culling and blending rules."""
import numpy as np

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)
FLOATS, F_DC, F_REST, OPACITY, SCALE, ROT = 62, 6, 9, 54, 55, 58


def fibonacci_directions(n):
    """(n, 3) float32: z_j = 1 - (2j + 1) / n, phi_j = j pi (3 - sqrt 5), in double, then rounded"""
    j = np.arange(n, dtype=np.float64)
    z = 1.0 - (2.0 * j + 1.0) / n
    phi = j * (np.pi * (3.0 - np.sqrt(5.0)))
    r = np.sqrt(np.maximum(0.0, 1.0 - z * z))
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1).astype(np.float32)


def sh_basis(d):
    """(n, 16) float64: 3DGS's basis (sh_utils.py eval_sh) at the directions d (n, 3), taken as they are"""
    d = np.asarray(d, np.float64)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    return np.stack([
        np.full_like(x, C0), -C1 * y, C1 * z, -C1 * x,
        C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy),
        C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
        C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy)], 1)


def weights(dirs, normal):
    """(D,) w_j = max(0, -d_j . n) for n != 0, else 1, in double from the fp32 values"""
    d = np.asarray(dirs, np.float64)
    n = np.asarray(normal, np.float64)
    if not n.any():
        return np.ones(d.shape[0])
    dn = (d[:, 0] * n[0] + d[:, 1] * n[1]) + d[:, 2] * n[2]
    return np.maximum(0.0, -dn)


PIVOT_RTOL = 1e-10


def cholesky(A):
    """lower factor of A by the right-looking rule, or None when a pivot is at most PIVOT_RTOL times A's largest
    diagonal entry (a rank-deficient system)"""
    A = np.array(A, np.float64)
    n = A.shape[0]
    tiny = PIVOT_RTOL * A.diagonal().max()
    if not A.diagonal().max() > 0:
        return None
    for k in range(n):
        if not A[k, k] > tiny:
            return None
        A[k, k] = np.sqrt(A[k, k])
        A[k + 1:, k] /= A[k, k]
        A[k + 1:, k + 1:] -= np.outer(A[k + 1:, k], A[k + 1:, k])
    return np.tril(A)


def fit(colors, dirs, normals, degree, ridge):
    """colors (P, D, 3) (the fp16 colours as numbers), dirs (D, 3) fp32, normals (P, 3) or None -> coefficients
    (P, 3, 16) float64, 0 above the degree, and all 0 where the system is rank-deficient (cholesky)"""
    colors = np.asarray(colors, np.float64)
    P, D = colors.shape[:2]
    nb = (degree + 1) ** 2
    Y = sh_basis(dirs)[:, :nb]
    out = np.zeros((P, 3, 16))
    for p in range(P):
        w = weights(dirs, np.zeros(3) if normals is None else normals[p])
        A = (Y * w[:, None]).T @ Y + ridge * w.sum() * np.eye(nb)
        b = (Y * w[:, None]).T @ (colors[p] - 0.5)
        Lf = cholesky(A)
        if Lf is not None:
            out[p, :, :nb] = np.linalg.solve(Lf.T, np.linalg.solve(Lf, b)).T
    return out


def sh_fields(coef):
    """(P, 3, 16) coefficients -> f_dc (P, 3), f_rest (P, 45) in the file's channel-major order"""
    coef = np.asarray(coef)
    return coef[:, :, 0], coef[:, :, 1:].reshape(coef.shape[0], 45)


def quaternion(n):
    """(w, x, y, z) float64 of the shortest arc taking +z to n / |n|; (0, 1, 0, 0) when that arc is a half turn"""
    n = np.asarray(n, np.float64)
    ln = np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])
    u = n / ln
    w, x, y = 1.0 + u[2], -u[1], u[0]
    nq = np.sqrt((w * w + x * x) + y * y)
    if nq == 0:
        return np.array([0.0, 1.0, 0.0, 0.0])
    return np.array([w / nq, x / nq, y / nq, 0.0])


def rotation(q):
    """3 x 3 rotation of a (w, x, y, z) quaternion, normalised first (3DGS's build_rotation)"""
    w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def geometry(points, normals, sigma, dist2, shape="disc", flatness=0.1):
    """every field but f_dc / f_rest of the (P, 62) splats, float64 (positions and normals as given): the scale rule,
    the quaternion and the opacity of stage 3"""
    points = np.asarray(points, np.float32)
    P = points.shape[0]
    normals = np.zeros((P, 3), np.float32) if normals is None else np.asarray(normals, np.float32)
    dist2 = np.asarray(dist2, np.float64).reshape(P, -1)
    sigma = np.asarray(sigma, np.float32)
    out = np.zeros((P, FLOATS))
    kk = min(dist2.shape[1], 3)
    for i in range(P):
        out[i, 0:3] = points[i]
        out[i, 3:6] = normals[i]
        m = 0.0
        for a in range(kk):
            m = m + dist2[i, a]
        if kk:
            m = m / kk
        s = np.sqrt(max(m, 1e-7))
        q, s_n = np.array([1.0, 0.0, 0.0, 0.0]), s
        if shape == "disc" and normals[i].any():
            q = quaternion(normals[i])
            s_n = np.float64(np.float32(flatness)) * s
        alpha = min(max(1.0 - np.exp(-np.float64(sigma[i]) * 2.0 * s), 0.01), 0.99)
        out[i, OPACITY] = np.log(alpha / (1.0 - alpha))
        out[i, SCALE:SCALE + 3] = np.log([s, s, s_n])
        out[i, ROT:ROT + 4] = q
    return out


def eval_color(splat, u):
    """one splat's colour (3,) along the unit direction u: max(0, SH + 0.5)"""
    y = sh_basis(np.asarray(u, np.float64)[None])[0]
    coef = np.concatenate([splat[F_DC:F_DC + 3, None], np.asarray(splat[F_REST:F_REST + 45]).reshape(3, 15)], 1)
    return np.maximum(coef @ y + 0.5, 0.0)


def rasterize(splats, pose, K, W, H, bg):
    """float64 brute force: per pixel, every splat whose tile rectangle holds the pixel's tile, in (depth, index)
    order, blended with the rasteriser's rules -> rgb (H, W, 3), opacity (H, W)"""
    splats = np.asarray(splats, np.float64)
    pose = np.asarray(pose, np.float64).reshape(3, 4)
    R, o = pose[:, :3], pose[:, 3]
    fx, fy, cx, cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
    gx, gy = (W + 15) // 16, (H + 15) // 16
    items = []
    for i, g in enumerate(splats):
        d = g[0:3] - o
        c = R.T @ d
        if not c[2] > 0.2:
            continue
        q = g[ROT:ROT + 4]
        if not np.linalg.norm(q) > 0:
            continue
        Rq = rotation(q)
        S = Rq @ np.diag(np.exp(g[SCALE:SCALE + 3]) ** 2) @ Rq.T
        limx, limy = 1.3 * (0.5 * W / fx), 1.3 * (0.5 * H / fy)
        tx = min(limx, max(-limx, c[0] / c[2])) * c[2]
        ty = min(limy, max(-limy, c[1] / c[2])) * c[2]
        J = np.array([[fx / c[2], 0, -fx * tx / c[2] ** 2], [0, fy / c[2], -fy * ty / c[2] ** 2]])
        T = J @ R.T
        cov = T @ S @ T.T + 0.3 * np.eye(2)
        det = cov[0, 0] * cov[1, 1] - cov[0, 1] ** 2
        if not det > 0:
            continue
        mid = 0.5 * (cov[0, 0] + cov[1, 1])
        lam = mid + np.sqrt(max(0.1, mid * mid - det))
        radius = np.ceil(3 * np.sqrt(lam))
        px, py = fx * c[0] / c[2] + cx - 0.5, fy * c[1] / c[2] + cy - 0.5
        rx0 = min(gx, max(0, int((px - radius) / 16)))
        ry0 = min(gy, max(0, int((py - radius) / 16)))
        rx1 = min(gx, max(0, int((px + radius + 15) / 16)))
        ry1 = min(gy, max(0, int((py + radius + 15) / 16)))
        if (rx1 - rx0) * (ry1 - ry0) == 0:
            continue
        conic = np.array([cov[1, 1], -cov[0, 1], cov[0, 0]]) / det
        op = 1.0 / (1.0 + np.exp(-g[OPACITY]))
        col = eval_color(g, d / np.linalg.norm(d))
        items.append((c[2], i, px, py, conic, op, col, (rx0, ry0, rx1, ry1)))
    items.sort(key=lambda t: (t[0], t[1]))
    ys, xs = np.mgrid[0:H, 0:W]
    xs, ys = xs.astype(np.float64), ys.astype(np.float64)
    tx_, ty_ = (xs // 16).astype(int), (ys // 16).astype(int)
    Tr = np.ones((H, W))
    C = np.zeros((H, W, 3))
    done = np.zeros((H, W), bool)
    for _, _, px, py, conic, op, col, (rx0, ry0, rx1, ry1) in items:
        inside = (tx_ >= rx0) & (tx_ < rx1) & (ty_ >= ry0) & (ty_ < ry1) & ~done
        dx, dy = px - xs, py - ys
        power = -0.5 * (conic[0] * dx * dx + conic[2] * dy * dy) - conic[1] * dx * dy
        alpha = np.minimum(0.99, op * np.exp(np.minimum(power, 0.0)))
        use = inside & (power <= 0) & (alpha >= 1 / 255)
        test = Tr * (1 - alpha)
        stop = use & (test < 1e-4)
        done |= stop
        use &= ~stop
        C += np.where(use[..., None], col[None, None, :] * (alpha * Tr)[..., None], 0.0)
        Tr = np.where(use, test, Tr)
    return C + Tr[..., None] * np.asarray(bg, np.float64), 1.0 - Tr
