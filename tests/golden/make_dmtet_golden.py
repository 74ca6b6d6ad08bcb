"""Generates tests/golden/ref_dmtet.npz by running the reference's own `marching_tets` and `sdf_reg_loss` (geometry/dmtet.py) on the CPU.

geometry/dmtet.py cannot be imported without a GPU: it imports the renderer and builds its lookup tables on "cuda" at import.  So this
script parses the file and evaluates, from its syntax tree, only `triangle_table`, `num_triangles_table`, `base_tet_edges`, `v_id`,
`sort_edges`, `map_uv`, `marching_tets` and `sdf_reg_loss`, with every device="cuda" argument turned into "cpu".  Nothing from the
reference is copied into this repository.

Grid: tests/golden/tets_32.npz (the reference's data/tets/32_tets.npz, 6 641 vertices, 30 136 tets).  SDF cases:
  init      the reference's initialisation rand - 0.1 (DMTetGeometry.__init__), seeded;
  sphere0   a sphere of radius 0.3, with about 20 % exact zeros and some -0.0;
  nonfinite the sphere with NaN, +-inf and +-3e38 entries.
The SDFs lie on lattices (2^-12 for the initialisation, 2^-16 for the sphere) so that the fixture compresses.  The positions are the
grid's vertices, as in DMTetGeometry at its initial deform = 0; the deformation (`deform_of`) and the upstream gradient of verts
(`d_verts_of`) are fixed patterns of the element index, computed, not stored.  Stored once: `uvs` as its shape, first rows and SHA-256
(`uvs_shape`, `uvs_head`, `uvs_sha256`: the full table is 0.97 MB and depends only on the tet count).  Per case, under "<case>/...": the
sdf, the outputs (verts; faces packed by `pack_faces`; uv_idx as the differences of its faces' tet ids, `uv_tet`; `unpack_faces` and
`unpack_uv_idx` expand them), the gradients of the upstream gradient with respect to pos and sdf, and sdf_reg_loss over the grid's edges (DMTetGeometry.all_edges) with the upstream gradient of the
loss and the resulting d sdf.  The gradient with respect to `deform` through getMesh's `verts + 2 / (2 * res) * tanh(deform)` does not
depend on the positions, only on d pos: generation checks that the reference's equals d pos x 2 / (2 res) x (1 - tanh(deform)^2) within
1e-6, and the tests check the product's against the same product of the stored d pos.  Everything stored is what the reference computed,
in a lossless encoding.
    python tests/golden/make_dmtet_golden.py
"""
import ast
import hashlib
import os

import numpy as np
import torch

REF = "/root/reference/geometry/dmtet.py"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "ref_dmtet.npz")
GRID = os.path.join(HERE, "tets_32.npz")
RES = 32
NAMES = ("triangle_table", "num_triangles_table", "base_tet_edges", "v_id", "sort_edges", "map_uv", "marching_tets", "sdf_reg_loss")


class _ToCpu(ast.NodeTransformer):
    def visit_Constant(self, node):
        return ast.copy_location(ast.Constant("cpu"), node) if node.value == "cuda" else node


def reference_functions(path=REF):
    """The NAMES of geometry/dmtet.py, evaluated on the CPU."""
    tree = ast.parse(open(path).read(), path)
    keep = []
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in NAMES:
            keep.append(node)
        elif isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id in NAMES for t in node.targets):
            keep.append(node)
    mod = ast.fix_missing_locations(_ToCpu().visit(ast.Module(body=keep, type_ignores=[])))
    ns = {"torch": torch, "np": np}
    exec(compile(mod, path, "exec"), ns)
    missing = [n for n in NAMES if n not in ns]
    assert not missing, missing
    return ns


def grid():
    t = np.load(GRID)
    return torch.tensor(t["vertices"]).float(), torch.tensor(t["indices"]).long()


def all_edges(indices):
    """DMTetGeometry.generate_edges: the unique sorted vertex pairs of the tets' six base edges."""
    e = indices[:, torch.tensor([0, 1, 0, 2, 0, 3, 1, 2, 1, 3, 2, 3])].reshape(-1, 2)
    return torch.unique(torch.sort(e, dim=1)[0], dim=0)


def uvs_digest(uvs):
    """SHA-256 of an fp32 [n,2] UV table's little-endian bytes, as a uint8 array."""
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(uvs, "<f4").tobytes()).digest(), np.uint8).copy()


def pack_uv_idx(uv_idx):
    """uv_idx [F,3] as the differences of its faces' tet ids (uv_idx[:,0] / 4), int32: each row is (4t, 4t+k+1, 4t+k+2) with k the face's
    index within its tet, so the tet ids determine it (a tet's second face follows its first)."""
    return np.diff(uv_idx[:, 0] // 4, prepend=0).astype(np.int32)


def unpack_uv_idx(uv_tet):
    t = np.cumsum(uv_tet.astype(np.int64))
    k = np.concatenate([[0], (t[1:] == t[:-1]).astype(np.int64)]) if t.size else t
    return np.stack([4 * t, 4 * t + k + 1, 4 * t + k + 2], -1)


def deform_of(V):
    """The deformation [V,3]: multiples of 1/32 in [-0.25, 0.25], a fixed pattern of the element index."""
    j = np.arange(3 * V, dtype=np.int64)
    return (((j * 7919) % 17 - 8) / 32).astype(np.float32).reshape(V, 3)


def d_verts_of(M):
    """The upstream gradient of verts [M,3]: multiples of 1/4 in [-1, 1], a fixed pattern of the element index."""
    j = np.arange(3 * M, dtype=np.int64)
    return (((j * 104729) % 9 - 4) / 4).astype(np.float32).reshape(M, 3)


def pack_faces(faces):
    """faces [F,3] as int16: the differences of the first column, then the other two columns relative to the first."""
    f = faces.astype(np.int64)
    out = np.stack([np.diff(f[:, 0], prepend=0), f[:, 1] - f[:, 0], f[:, 2] - f[:, 0]], -1)
    assert np.abs(out).max(initial=0) < 2 ** 15
    return out.astype(np.int16)


def unpack_faces(packed):
    p = packed.astype(np.int64)
    c0 = np.cumsum(p[:, 0])
    return np.stack([c0, c0 + p[:, 1], c0 + p[:, 2]], -1)


def rel_l2(a, b):
    """Relative L2 over the entries finite in both."""
    f = np.isfinite(a) & np.isfinite(b)
    return np.linalg.norm(a[f] - b[f]) / max(np.linalg.norm(b[f]), 1e-30)


def sdf_cases(verts):
    V = verts.shape[0]
    g = torch.Generator().manual_seed(2024)
    init = torch.randint(0, 4096, (V,), generator=g).float() / 4096 - 0.1     # rand - 0.1 on a 2^-12 lattice
    sphere = torch.round((0.3 - verts.norm(dim=1)) * 65536) / 65536
    sphere0 = sphere.clone()
    pick = torch.rand(V, generator=g)
    sphere0[pick < 0.2] = 0.0
    sphere0[(pick >= 0.2) & (pick < 0.23)] = -0.0
    nonfinite = sphere.clone()
    for value, frac in ((float("nan"), 0.01), (float("inf"), 0.01), (-float("inf"), 0.01), (3e38, 0.01), (-3e38, 0.01)):
        nonfinite[torch.randperm(V, generator=g)[:int(frac * V)]] = value
    return {"init": init, "sphere0": sphere0, "nonfinite": nonfinite}


def generate():
    """The fixture's arrays.  Runs on one CPU thread: autograd's scatter-adds into pos and sdf then sum in one fixed order."""
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        return _generate()
    finally:
        torch.set_num_threads(threads)


def _generate():
    ns = reference_functions()
    verts, indices = grid()
    edges = all_edges(indices)
    g = torch.Generator().manual_seed(99)
    deform0 = torch.from_numpy(deform_of(verts.shape[0]))
    d = {}
    for name, sdf0 in sdf_cases(verts).items():
        pos = verts.clone().requires_grad_(True)
        sdf = sdf0.clone().requires_grad_(True)
        out_v, faces, uvs, uv_idx = ns["marching_tets"](pos, sdf, indices)
        gv = torch.from_numpy(d_verts_of(out_v.shape[0]))
        d_pos, d_sdf = torch.autograd.grad(out_v, (pos, sdf), gv)
        # through getMesh's deformation, the chain rule applied to d pos
        deform = deform0.clone().requires_grad_(True)
        out_d = ns["marching_tets"](verts + 2 / (RES * 2) * torch.tanh(deform), sdf0.clone(), indices)[0]
        d_deform, = torch.autograd.grad(out_d, (deform,), gv)
        t = np.tanh(deform0.numpy().astype(np.float64))
        assert rel_l2(d_pos.numpy() * (2 / (2 * RES)) * (1 - t * t), d_deform.numpy()) <= 1e-6
        sdf_r = sdf0.clone().requires_grad_(True)
        reg = ns["sdf_reg_loss"](sdf_r, edges)
        d_loss = torch.rand((), generator=g) + 0.5
        d_reg, = torch.autograd.grad(reg, (sdf_r,), d_loss)
        uv_tet = pack_uv_idx(uv_idx.numpy())
        assert np.array_equal(unpack_uv_idx(uv_tet), uv_idx.numpy())
        assert np.array_equal(unpack_faces(pack_faces(faces.numpy())), faces.numpy())
        d.update({name + "/sdf": sdf0.numpy(), name + "/verts": out_v.detach().numpy(), name + "/faces": pack_faces(faces.numpy()),
                  name + "/uv_tet": uv_tet, name + "/d_pos": d_pos.numpy(),
                  name + "/d_sdf": d_sdf.numpy(), name + "/reg_loss": reg.detach().numpy(),
                  name + "/reg_d_loss": d_loss.numpy(), name + "/reg_d_sdf": d_reg.numpy()})
        d.update({"uvs_shape": np.array(uvs.shape, np.int64), "uvs_head": uvs[:64].numpy(), "uvs_sha256": uvs_digest(uvs.numpy())})
    return d


if __name__ == "__main__":
    d = generate()
    np.savez_compressed(OUT, **d)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", ", ".join("%s %d verts %d faces" % (c, len(d[c + "/verts"]), len(d[c + "/faces"]))
                                                                   for c in ("init", "sphere0", "nonfinite")))
