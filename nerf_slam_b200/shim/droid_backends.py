"""`import droid_backends` of the reference (networks/modules/corr.py:4, visual_frontend.py:24) -> the sm_90a module"""
from nerf_slam_b200.droid_backends import *  # noqa: F401,F403
from nerf_slam_b200.droid_backends import (altcorr_forward, ba, corr_index_forward, depth_filter, frame_distance, iproj,  # noqa: F401
                                           projmap, reduced_camera_matrix, solve_depth, solve_poses)
