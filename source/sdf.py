"""source.sdf -> points2surf_b200.sdf (get_voxel_centers_grid_smaller_pc, implicit_surface_to_mesh[_file|_directory],
get_query_pts_for_mesh, get_signed_distance, ...)."""
from points2surf_b200.sdf import *  # noqa: F401,F403
from points2surf_b200.sdf import (get_voxel_centers_grid_smaller_pc, model_space_to_volume_space, implicit_surface_to_mesh,  # noqa: F401
                                  implicit_surface_to_mesh_file, implicit_surface_to_mesh_directory, visualize_query_points,
                                  get_query_pts_for_mesh, get_signed_distance)
