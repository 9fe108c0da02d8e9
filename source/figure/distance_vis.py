"""source.figure.distance_vis -> points2surf_b200.figure.distance_vis (make_distance_comparison, ...)."""
from points2surf_b200.figure.distance_vis import *  # noqa: F401,F403
from points2surf_b200.figure.distance_vis import (get_normalization_target, visualize_mesh_with_distances,  # noqa: F401
                                                  make_distance_comparison, main)
