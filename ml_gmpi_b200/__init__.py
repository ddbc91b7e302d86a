"""H100-native multiplane-image renderer: drop-in for the render path of apple/ml-gmpi
(gmpi/core/mpi.py MPI.forward + homography, driven by MPIRenderer.render)."""
from . import _lib  # noqa: F401
from ._build import build_library  # noqa: F401
from .mpi import (MPI, MPIOutOfPlaneError, Occupancy, TrainPlan, build_occupancy, check_range, expand_factored,  # noqa: F401
                  render_frames, render_views, render_views_factored, train_plan, unorm8_to_float)

__all__ = ["MPI", "MPIOutOfPlaneError", "render_views", "render_views_factored", "render_frames", "expand_factored", "check_range",
           "build_library", "build_occupancy", "Occupancy", "unorm8_to_float", "train_plan", "TrainPlan"]
