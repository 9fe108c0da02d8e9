"""source/figure/distance_vis.py: colour every vertex of a reconstruction by its distance to the ground-truth mesh
(get_closest_distance_batched on the GPU).  Per reconstruction <mesh> it writes
  <mesh>_vis.ply    the reconstruction with per-vertex colours;
  <mesh>_stats.txt  the reference's one-line statistics, same text;
  <mesh>_dist.npy   the distances [V] float64 themselves, so the colours are never the only record.
Deviation: the colours come from COLOR_RAMP below (blue at distance 0, green at half the normalisation target, yellow at
and beyond it), not from the reference's parula table."""
import numpy as np

from .. import mesh_io
from ..point_cloud import get_closest_distance_batched

# piecewise-linear ramp through blue (0), green (0.5) and yellow (1), 256 entries of RGB in [0, 1]
_RAMP_ANCHORS = np.array([[0.2, 0.2, 0.9], [0.1, 0.7, 0.4], [1.0, 0.9, 0.1]])
COLOR_RAMP = np.stack([np.interp(np.linspace(0.0, 1.0, 256), [0.0, 0.5, 1.0], _RAMP_ANCHORS[:, k]) for k in range(3)], 1)


def get_normalization_target(distances: list, cut_percentil=0.9):
    """distance_vis.py:12-19: the distance at index int(n * cut_percentil) of the sorted concatenation (the largest one
    when cut_percentil is None or >= 1)."""
    dist_concat_sorted = np.sort(np.concatenate(distances, axis=0))
    if cut_percentil is not None and cut_percentil < 1.0:
        return dist_concat_sorted[int(dist_concat_sorted.shape[0] * cut_percentil)]
    return dist_concat_sorted[-1]


def distance_colors(dist_per_vertex, normalize_to):
    """RGB [V,3] in [0, 1]: COLOR_RAMP at int(dist / normalize_to * 255), clamped to the last entry (distance_vis.py:25-30
    with COLOR_RAMP for the parula table).  A target of 0 colours everything as distance 0."""
    d = np.asarray(dist_per_vertex, np.float64)
    norm = d / normalize_to if normalize_to > 0 else np.zeros_like(d)
    idx = (norm * (COLOR_RAMP.shape[0] - 1)).astype(np.int32)
    idx[idx >= COLOR_RAMP.shape[0]] = COLOR_RAMP.shape[0] - 1
    return COLOR_RAMP[idx]


def visualize_mesh_with_distances(mesh_file: str, mesh, dist_per_vertex: np.ndarray, normalize_to: float,
                                  cut_percentil=0.9):
    """distance_vis.py:22-44: writes <mesh_file>_vis.ply, <mesh_file>_stats.txt and <mesh_file>_dist.npy.
    `mesh`: anything with .vertices / .faces, or a (vertices, faces) pair."""
    verts, faces = (mesh.vertices, mesh.faces) if hasattr(mesh, 'vertices') else mesh
    mesh_io.write_ply(mesh_file + '_vis.ply', verts, faces, colors=distance_colors(dist_per_vertex, normalize_to))
    np.save(mesh_file + '_dist.npy', np.asarray(dist_per_vertex))
    with open(mesh_file + '_stats.txt', 'w+') as stats_file:
        stats_file.write(
            'Distance from reconstructed mesh vertex to nearest sample on GT mesh, '
            'Min={}, Max={}, Mean={}, normalized to {}, cut percentil {}'.format(
                np.min(dist_per_vertex), np.max(dist_per_vertex), np.mean(dist_per_vertex), normalize_to, cut_percentil))


def make_distance_comparison(in_file_rec_meshes: list, in_file_gt_mesh, cut_percentil=0.9, batch_size=1000):
    """distance_vis.py:47-75: the distance of every vertex of every reconstruction to the ground-truth mesh
    (in_file_gt_mesh: one file for all, or one per reconstruction), normalised to the common target of
    get_normalization_target, written next to each reconstruction."""
    meshes_rec = [mesh_io.read_mesh(f) for f in in_file_rec_meshes]
    if isinstance(in_file_gt_mesh, str):
        mesh_gt = mesh_io.read_mesh(in_file_gt_mesh)
        meshes_gt = [mesh_gt] * len(meshes_rec)
    elif isinstance(in_file_gt_mesh, list):
        meshes_gt = [mesh_io.read_mesh(f) for f in in_file_gt_mesh]
    else:
        raise ValueError('Not implemented!')
    vertices_rec_dists = [get_closest_distance_batched(mesh_rec[0], meshes_gt[mi], batch_size)[1]
                          for mi, mesh_rec in enumerate(meshes_rec)]
    normalize_to = get_normalization_target(vertices_rec_dists, cut_percentil=cut_percentil)
    for fi, f in enumerate(in_file_rec_meshes):
        visualize_mesh_with_distances(f, meshes_rec[fi], dist_per_vertex=vertices_rec_dists[fi],
                                      normalize_to=normalize_to, cut_percentil=cut_percentil)


def main(in_file_rec_meshes: list, in_file_gt_mesh, cut_percentile=0.9, batch_size=1000):
    print('Visualize distances of {} to {}'.format(in_file_rec_meshes, in_file_gt_mesh))
    make_distance_comparison(in_file_rec_meshes=in_file_rec_meshes, in_file_gt_mesh=in_file_gt_mesh,
                             cut_percentil=cut_percentile, batch_size=batch_size)
