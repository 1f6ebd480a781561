"""CPU: the sweeps' numpy sources (stitcher._sweep_sources).  A source that is not C-contiguous is read through a
contiguous copy, and that copy is what the caller gets back to hold while the sweep runs: the pointers the sweep
hands to the library are those of the returned arrays, which equal the sources."""
import numpy as np

from openpano_b200.capi import SRC_F32_HOST, SRC_RGB8_HOST
from openpano_b200.stitcher import _sweep_sources


def test_copies_of_views_are_returned_to_the_caller():
    rng = np.random.RandomState(3)
    rgb = rng.randint(0, 256, (30, 40, 4)).astype(np.uint8)[..., :3]        # every fourth byte skipped
    grey = rng.randint(0, 256, (60, 40)).astype(np.uint8)[::2]              # every other row
    dense = rng.randint(0, 256, (30, 40, 3)).astype(np.uint8)
    kind, formats, shapes, srcs, nbytes = _sweep_sources([rgb, dense, grey], 3, None, None, None, ["rgb", "rgb", "grey"])
    assert kind == SRC_RGB8_HOST and shapes == [(30, 40)] * 3
    for a, s in zip([rgb, dense, grey], srcs):
        assert isinstance(s, np.ndarray) and s.flags.c_contiguous and np.array_equal(s, a)
    assert srcs[1] is dense                                                 # a contiguous source is read in place
    assert nbytes == [s.nbytes for s in srcs]
    f32 = rng.rand(30, 40, 3).astype(np.float32)[:, ::-1]
    kind, formats, shapes, srcs, _ = _sweep_sources([f32], 1, None, None, None, None)
    assert kind == SRC_F32_HOST and formats == [3] and srcs[0].flags.c_contiguous and np.array_equal(srcs[0], f32)


def test_pointer_sources_pass_through():
    kind, formats, shapes, srcs, nbytes = _sweep_sources([1234, 5678], 2, SRC_RGB8_HOST, [3, 1], [(4, 5), (6, 7)], None)
    assert srcs == [1234, 5678] and nbytes == [60, 42] and formats == [3, 1]
