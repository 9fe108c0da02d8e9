"""Figures of the reference's source/figure/ (distance_vis)."""
