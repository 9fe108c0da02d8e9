"""source.base.point_cloud -> points2surf_b200.point_cloud (get_closest_distance_batched, write_xyz)."""
from points2surf_b200.point_cloud import get_closest_distance_batched, write_xyz  # noqa: F401
