"""Tet grids and SDFs for the DMTet tests: the reference's 32 grid (tests/golden/tets_32.npz) and procedural Kuhn grids."""
import importlib.util
import itertools
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def grid32():
    """(vertices [6641,3] fp32, indices [30136,4] int64) of the reference's 32 grid."""
    t = np.load(os.path.join(GOLDEN, "tets_32.npz"))
    return t["vertices"].astype(np.float32), t["indices"].astype(np.int64)


def kuhn_grid(n, lo=-0.5, hi=0.5):
    """(vertices [(n+1)^3, 3] fp32, tets [6 n^3, 4] int64): each of the n^3 cubes split into the 6 tets along the axis-ordered paths from
    its low corner to its high corner."""
    r = np.arange(n + 1)
    k, j, i = np.meshgrid(r, r, r, indexing="ij")
    verts = (np.stack([i, j, k], -1).reshape(-1, 3) / n * (hi - lo) + lo).astype(np.float32)
    c = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 3)[:, ::-1]   # (i, j, k), i fastest
    vid = lambda p: (p[:, 2] * (n + 1) + p[:, 1]) * (n + 1) + p[:, 0]
    tets = []
    for perm in itertools.permutations(range(3)):
        p, path = c.copy(), [vid(c)]
        for ax in perm:
            p = p.copy()
            p[:, ax] += 1
            path.append(vid(p))
        tets.append(np.stack(path, -1))
    return verts, np.stack(tets, 1).reshape(-1, 4).astype(np.int64)


def ref_init_sdf(V, seed=0):
    """DMTetGeometry's initialisation rand - 0.1 (a large, noisy surface)."""
    import torch
    return (torch.rand(V, generator=torch.Generator().manual_seed(seed)) - 0.1).numpy()


def sphere_sdf(verts, radius=0.3):
    return (radius - np.linalg.norm(verts.astype(np.float64), axis=1)).astype(np.float32)


def ref_all_edges(indices):
    """DMTetGeometry.all_edges: the unique (min, max) vertex pairs of the tets' six base edges, sorted lexicographically."""
    pairs = np.sort(np.asarray(indices)[:, [0, 1, 0, 2, 0, 3, 1, 2, 1, 3, 2, 3]].reshape(-1, 2), 1)
    return np.unique(pairs, axis=0).astype(np.int32)


def golden_codec():
    """tests/golden/make_dmtet_golden.py: the fixture's encodings and its computed inputs."""
    spec = importlib.util.spec_from_file_location("make_dmtet_golden", os.path.join(GOLDEN, "make_dmtet_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_dmtet_golden():
    """tests/golden/ref_dmtet.npz decoded: {case: {sdf, verts, faces, uv_idx, d_verts, d_pos, d_sdf, reg_loss, reg_d_loss, reg_d_sdf}} plus
    "deform", "uvs_shape", "uvs_head", "uvs_sha256" and the "codec" module."""
    mk = golden_codec()
    z = dict(np.load(os.path.join(GOLDEN, "ref_dmtet.npz")))
    V = grid32()[0].shape[0]
    out = {"deform": mk.deform_of(V), "uvs_shape": tuple(z["uvs_shape"]), "uvs_head": z["uvs_head"], "uvs_sha256": z["uvs_sha256"], "codec": mk}
    for case in ("init", "sphere0", "nonfinite"):
        c = {k.split("/", 1)[1]: v for k, v in z.items() if k.startswith(case + "/")}
        c["faces"] = mk.unpack_faces(c.pop("faces"))
        c["uv_idx"] = mk.unpack_uv_idx(c.pop("uv_tet"))
        c["d_verts"] = mk.d_verts_of(c["verts"].shape[0])
        out[case] = c
    return out
