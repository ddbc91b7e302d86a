"""Drop-in boundary: the host-side mirrors must accept exactly what the reference's callers pass (SURVEY.md 8b).
The reference's signatures are recorded in tests/golden/reference_signatures.json (oracle/make_golden_signatures.py)."""
import inspect

from make_golden_signatures import params as _params
from testlib import reference_signatures


def test_mpi_signatures():
    ref = reference_signatures()["MPI"]
    import ml_gmpi_b200 as g
    ours, theirs = _params(g.MPI.forward), ref["forward"]
    assert ours == theirs                                            # keyword-only, same names, same defaults
    assert _params(g.MPI.check_shapes) == ref["check_shapes"]
    init_ref = ref["__init__"]
    init_ours = _params(g.MPI.__init__)
    assert init_ours[: len(init_ref)] == init_ref                    # ours adds the optional `validate` after align_corners


def test_renderer_signatures():
    ref = reference_signatures()["MPIRenderer"]
    from ml_gmpi_b200.renderer import MPIRenderer
    for name in ("render", "sample_cam_poses", "set_cam", "compute_mpi_spatial_volume"):
        assert _params(getattr(MPIRenderer, name)) == ref[name], name
    ref_init = ref["__init__"]
    ours_init = _params(MPIRenderer.__init__)
    assert ours_init[: len(ref_init)] == ref_init                    # ours adds the optional `validate`


def test_reference_call_site_binds():
    """mpi_renderer.py:451-461 calls self.mpi(batch_rgba=..., ..., c2w_mat=..., sphere_c=...): must bind to our forward."""
    import ml_gmpi_b200 as g
    sig = inspect.signature(g.MPI.forward)
    sig.bind(None, batch_rgba=1, batch_dhw=2, batch_ray_dir=3, batch_eye_pos=4, batch_z_dir=5, separate_background=None,
             assert_not_out_of_last_plane=True, c2w_mat=6, sphere_c=7)
