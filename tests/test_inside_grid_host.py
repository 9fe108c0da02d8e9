"""The solid voxelisation's CPU oracle (oracle/inside_oracle.py) and the host side of make_dataset --gt_recon.

- The oracle's parity against the float64 winding-number sign of oracle/mesh_sdf_oracle.py at voxels farther than 1e-5
  from the surface, on an icosphere, a torus and the three abc_minimal meshes, at res 16-32.  The winding oracle costs
  ~1 us per (query, face) pair, so it is asked at every voxel next to a change of the oracle's flag (where a wrong rule
  shows first) and at a seeded sample of the others, at most 5e6 pairs per mesh.
- An axis-aligned box and an octahedron whose corners and projected edges lie exactly on column centres: every column is
  crossed an even number of times and the inside set is the one geometry and the tie rule give.
- The grid-target stage (05_query_pts_grid, 05_query_dist_grid) on a tiny dataset, with the two device calls replaced by
  CPU oracles: file names, dtypes, the clean-up rules of the query stage, and the mtime rule."""
import os
import time

import numpy as np
import pytest

import inside_cases as ic
from oracle import inside_oracle as io
from oracle import mesh_sdf_oracle as msdf
from oracle import p2s_oracle as orc
from points2surf_b200 import make_dataset, mesh_io, sdf

WINDING_CASES = [('sphere', 32), ('torus', 24), ('abc0', 16), ('abc1', 20), ('abc2', 32)]


def _voxel_centres(res, idx):
    c = io.centres(res)
    ix, rem = np.divmod(idx, res * res)
    iy, iz = np.divmod(rem, res)
    return np.stack([c[ix], c[iy], c[iz]], 1)


@pytest.mark.parametrize('name,res', WINDING_CASES)
def test_oracle_parity_matches_winding_number_sign(name, res):
    v, f = ic.closed_cases()[name]
    inside, cross = io.inside_grid(v, f, res)
    assert (cross % 2 == 0).all()
    flag = inside.astype(bool)
    shell = np.zeros_like(flag)
    for ax in range(3):
        d = np.diff(flag, axis=ax)
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, -1), slice(1, None)
        shell[tuple(lo)] |= d
        shell[tuple(hi)] |= d
    rng = np.random.RandomState(res)
    idx = np.flatnonzero(shell.reshape(-1))
    others = np.flatnonzero(~shell.reshape(-1))
    cap = int(5e6 // len(f))
    if len(idx) > cap - 200:
        idx = rng.choice(idx, cap - 200, replace=False)
    idx = np.concatenate([idx, rng.choice(others, min(200, len(others)), replace=False)])
    d, _, w = msdf.mesh_signed_distance(v, f, _voxel_centres(res, idx))
    far = np.abs(d) > 1e-5
    got = flag.reshape(-1)[idx]
    assert far.sum() > 0.9 * len(idx)
    # the crossing parity is the winding number mod 2, the distance's sign where the winding number is 0 or 1 (abc0 is two
    # overlapping closed components: w = 2 in the overlap, positive distance, even parity)
    wr = np.round(w)
    assert np.abs(w - wr)[far].max() < 1e-3
    assert (got == (wr % 2 == 1))[far].all()
    simple = far & ((wr == 0) | (wr == 1))
    bad = int((got != (d > 0))[simple].sum())
    assert bad == 0, (name, res, bad, len(idx))
    assert got.any() and not got.all()


@pytest.mark.parametrize('kind', ['box', 'octahedron'])
def test_lattice_meshes_cross_every_column_evenly_and_give_the_geometric_inside_set(kind):
    v, f = getattr(ic, kind)()
    inside, cross = io.inside_grid(v, f, ic.LATTICE_RES)
    assert (cross % 2 == 0).all()
    assert cross.max() == 2
    want = getattr(ic, kind + '_inside')()
    assert want.sum() > 40
    assert np.array_equal(inside, want), int((inside != want).sum())


def test_lattice_columns_on_projected_edges_and_vertices_are_taken_once():
    # the octahedron's apexes project onto column (7, 7), its apex edges onto row / column 7, its equator edges onto
    # diagonals of centres: each such column is crossed by exactly one upper and one lower face
    v, f = ic.octahedron()
    col, _ = io.crossings(v[:, :], f, ic.LATTICE_RES)
    cross = np.bincount(col, minlength=ic.LATTICE_RES ** 2).reshape(ic.LATTICE_RES, ic.LATTICE_RES)
    r = np.abs(np.arange(16)[:, None] - 7) + np.abs(np.arange(16)[None, :] - 7)
    assert (cross[r < 4] == 2).all() and (cross[r > 4] == 0).all()
    assert set(np.unique(cross[r == 4])) <= {0, 2}


def test_oracle_rejects_out_of_range_input():
    v, f = ic.box()
    with pytest.raises(ValueError, match='face index'):
        io.inside_grid(v, f + 100, 16)
    bad = v.copy()
    bad[0, 0] = 16.0
    with pytest.raises(ValueError, match='16'):
        io.inside_grid(bad, f, 16)


def test_mesh_is_closed():
    v, f = ic.icosphere(level=2)
    assert make_dataset.mesh_is_closed(f)
    assert not make_dataset.mesh_is_closed(f[1:])                       # a deleted face: three boundary edges
    flipped = f.copy()
    flipped[0] = flipped[0, ::-1]
    assert not make_dataset.mesh_is_closed(flipped)                     # inconsistent orientation
    assert not make_dataset.mesh_is_closed(np.concatenate([f, f[:1]]))  # an edge in three faces
    assert not make_dataset.mesh_is_closed(np.zeros((0, 3), np.int32))


# ------------------------------------------------------------------ the grid-target stage on the CPU
def _cpu_grid(pts, res, eps):
    return orc.query_grid(pts.astype(np.float32), res, eps).astype(np.float32)


def _cpu_sdf(mesh, query, batch=1000):
    v, f = mesh
    d = msdf.mesh_signed_distance(v, f, np.asarray(query, np.float32))[0]
    d[:3] = [np.nan, np.inf, -np.inf]          # the clean-up rules get every case
    d[3], d[4] = 2.5, -3.0
    return d


def test_grid_target_stage_layout_cleanup_and_mtime_rule(tmp_path, monkeypatch):
    monkeypatch.setattr(sdf, 'get_voxel_centers_grid_smaller_pc', _cpu_grid)
    monkeypatch.setattr(sdf, 'get_signed_distance', _cpu_sdf)
    root = tmp_path / 'ds'
    for d in ('03_meshes', '04_pts'):
        (root / d).mkdir(parents=True)
    cases = {'sphere': ic.icosphere(level=2), 'box': ic.box(), 'nomesh': ic.octahedron()}
    rng = np.random.RandomState(0)
    for name, (v, f) in cases.items():
        if name != 'nomesh':
            mesh_io.write_ply(str(root / '03_meshes' / (name + '.ply')), v, f)
        pts = v[rng.randint(0, len(v), 200)]
        np.save(str(root / '04_pts' / (name + '.xyz.npy')), np.concatenate([pts, np.zeros_like(pts)], 1))
    args = (str(tmp_path), 'ds', '04_pts', '03_meshes', '05_query_pts_grid', '05_query_dist_grid', 16, 3)
    make_dataset.get_query_pts_dist_grid(*args)
    assert sorted(os.listdir(root / '05_query_pts_grid')) == ['box.xyz.npy', 'sphere.xyz.npy']
    assert sorted(os.listdir(root / '05_query_dist_grid')) == ['box.xyz.npy', 'sphere.xyz.npy']
    assert not (root / '05_patch_ids_grid').exists()
    for name in ('sphere', 'box'):
        q = np.load(str(root / '05_query_pts_grid' / (name + '.xyz.npy')))
        d = np.load(str(root / '05_query_dist_grid' / (name + '.xyz.npy')))
        pts = np.load(str(root / '04_pts' / (name + '.xyz.npy')))[:, :3]
        assert q.dtype == np.float32 and d.dtype == np.float32 and q.shape == (len(d), 3)
        assert np.array_equal(q, _cpu_grid(pts, 16, 3))
        want = msdf.mesh_signed_distance(*cases[name], q)[0]
        assert d[:5].tolist() == [0.0, 1.0, 1.0, 1.0, -1.0]       # NaN -> 0, either infinity -> 1, clipped
        assert np.array_equal(d[5:], np.clip(want[5:], -1, 1).astype(np.float32))
    # outputs newer than both inputs are kept; a newer input (the mesh or the points) rewrites its shape only
    files = {p: os.path.getmtime(p) for p in (root / '05_query_pts_grid').iterdir()}
    files.update({p: os.path.getmtime(p) for p in (root / '05_query_dist_grid').iterdir()})
    time.sleep(0.05)
    make_dataset.get_query_pts_dist_grid(*args)
    assert all(os.path.getmtime(p) == t for p, t in files.items())
    later = max(files.values()) + 10
    os.utime(str(root / '03_meshes' / 'box.ply'), (later, later))
    make_dataset.get_query_pts_dist_grid(*args)
    for p, t in files.items():
        assert (os.path.getmtime(p) != t) == (p.name == 'box.xyz.npy'), p
