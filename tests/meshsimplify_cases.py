"""Small meshes for the decimation tests (DESIGN.md §6g): height fields, fans, strips and non-manifold soups."""
import numpy as np


def grid(nx, ny, seed=0, jitter=0.3, z_noise=0.01, spacing=0.01, z0=None):
    """(nx x ny) vertex grid, two triangles per cell; z = z0 exactly when z0 is given (a planar grid)."""
    rng = np.random.default_rng(seed)
    X, Y = np.meshgrid(np.arange(nx, dtype=np.float64), np.arange(ny, dtype=np.float64), indexing="xy")
    X = X + rng.uniform(-jitter, jitter, X.shape) * (X > 0) * (X < nx - 1)
    Y = Y + rng.uniform(-jitter, jitter, Y.shape) * (Y > 0) * (Y < ny - 1)
    Z = np.full(X.shape, z0) if z0 is not None else rng.normal(0, z_noise, X.shape) / spacing + 0.3 * np.sin(X * 0.7) * np.cos(Y * 0.5)
    xyz = (np.stack([X, Y, Z], -1).reshape(-1, 3) * spacing).astype(np.float32)
    if z0 is not None:
        xyz[:, 2] = np.float32(z0)
    i = np.arange(nx * ny).reshape(ny, nx)
    a, b, c, d = i[:-1, :-1].ravel(), i[:-1, 1:].ravel(), i[1:, :-1].ravel(), i[1:, 1:].ravel()
    tri = np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)]).astype(np.uint32)
    return xyz, tri


def fan(n, seed=0, radius=1.0):
    """hub vertex 0 and a closed ring of n rim vertices: n triangles around one hub"""
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = radius * rng.uniform(0.8, 1.2, n)
    rim = np.stack([r * np.cos(t), r * np.sin(t), rng.normal(0, 0.02, n)], 1)
    xyz = np.vstack([[0.0, 0.0, 0.1], rim]).astype(np.float32)
    k = np.arange(n)
    tri = np.stack([np.zeros(n, np.int64), 1 + k, 1 + (k + 1) % n], 1).astype(np.uint32)
    return xyz, tri


def strip(n, seed=0):
    """a triangle strip of n triangles over n + 2 vertices"""
    rng = np.random.default_rng(seed)
    k = np.arange(n + 2)
    xyz = np.stack([k // 2 * 0.01, (k % 2) * 0.012, rng.normal(0, 0.001, n + 2)], 1).astype(np.float32)
    tri = np.stack([k[:-2], k[1:-1], k[2:]], 1).astype(np.uint32)
    tri[1::2] = tri[1::2][:, [1, 0, 2]]
    return xyz, tri


def soup(nV, nF, seed=0):
    """random faces over few vertices: non-manifold edges, duplicate, flipped and degenerate faces"""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-1, 1, (nV, 3)).astype(np.float32)
    tri = rng.integers(0, nV, (nF, 3)).astype(np.uint32)
    tri[::7, 1] = tri[::7, 0]                                      # degenerate: a repeated corner
    tri = np.vstack([tri, tri[::5], tri[::6, ::-1]])               # duplicates, flipped duplicates
    return xyz, tri
