"""The CUDA frame against the reference renderer's own compute shaders run on the CPU (oracle/_ref/libgsref.so, see
tests/test_ref_shaders.py), directly rather than through the oracle: MODE_EXACT at tile-cull levels 0, 1 and 2 against
the reference frame with the shared-definition exp, and at level 0 every debug buffer the two frames share."""
import numpy as np
import pytest

from test_ref_shaders import case, check_attr, same

pytestmark = pytest.mark.gpu

CASES = ["edge/axis640", "edge/rotated_odd", "edge/near_plane", "scale/rotated_odd", "c1/odd_size", "golden/c1_small"]


@pytest.fixture(scope="module")
def ref():
    import ref_shaders

    try:
        ref_shaders.load()
    except (RuntimeError, OSError) as e:
        pytest.fail(str(e), pytrace=False)
    return ref_shaders


@pytest.mark.parametrize("name", CASES)
def test_cuda_frame_equals_reference_shaders(gs, ref, name):
    vtx, u = case(name)
    ref.set_exp_mode(1)
    try:
        rf = ref.render_frame(vtx, u)
    finally:
        ref.set_exp_mode(0)
    c = gs.Context(0)
    try:
        c.set_mode(gs.MODE_EXACT)
        c.set_debug(True)
        c.upload(vtx)
        for level in (0, 1, 2):
            c.set_tile_cull(level)
            img = c.render(u, gs.FORMAT_RGBA32F)
            assert same(img, rf["rgba"]), (name, level)
            if level == 0:
                assert c.stats().num_instances == rf["m"], name
                assert same(c.download(gs.BUF_COV3D), ref.cov3d(vtx)), name
                check_attr(c.download(gs.BUF_ATTR), c.download(gs.BUF_TILES_OVERLAP), rf["attr"], rf["tiles"], name)
                assert np.array_equal(c.download(gs.BUF_PREFIX_SUM), rf["scan"]), name
                assert np.array_equal(c.download(gs.BUF_KEYS_SORTED), rf["keys"]), name
                assert np.array_equal(c.download(gs.BUF_VALS_SORTED), rf["vals"]), name
                assert np.array_equal(c.download(gs.BUF_TILE_BOUNDARY), rf["ranges"]), name
    finally:
        c.close()
