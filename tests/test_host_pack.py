"""CPU: the ragged-batch pack every engine wrapper hands the library, and the per-stream split of its results."""
import numpy as np
import pytest

from whisperlivekit_b200._lib import pack, split


@pytest.mark.parametrize("offs_dtype", [np.int32, np.int64])
@pytest.mark.parametrize("shape", [(), (3,)])
def test_pack_split_round_trip(offs_dtype, shape):
    rng = np.random.default_rng(0)
    lens = [0, 4, 0, 1, 7, 0]
    parts = [rng.standard_normal((n, *shape)).astype(np.float64) for n in lens]
    flat, offs = pack(parts, np.float32, shape, offs_dtype)
    assert offs.dtype == offs_dtype and offs.shape == (len(lens) + 1,)
    assert offs.tolist() == [0] + np.cumsum(lens).tolist()
    assert flat.dtype == np.float32 and flat.flags.c_contiguous and flat.shape == (sum(lens), *shape)
    back = split(flat, offs)
    assert len(back) == len(parts)
    for got, want in zip(back, parts):
        assert got.shape == want.shape
        np.testing.assert_array_equal(got, want.astype(np.float32))
    back[1][:] = 0                                              # copies: the packed rows are untouched
    assert flat[offs[1]: offs[2]].any()


@pytest.mark.parametrize("parts", [[], [[], ()], [np.zeros((0, 3))]], ids=["no-streams", "empty-streams", "empty-rows"])
def test_pack_without_rows_gives_one_zero_row(parts):
    shape = (3,) if any(np.ndim(p) == 2 for p in parts) else ()
    flat, offs = pack(parts, np.int32, shape, np.int64)
    assert flat.shape == (1, *shape) and flat.dtype == np.int32 and not flat.any()
    assert offs.tolist() == [0] * (len(parts) + 1)
    assert [p.shape for p in split(flat, offs)] == [(0, *shape)] * len(parts)


def test_pack_flattens_to_the_row_shape():
    """Token lists become one int32 row each; audio of whole 2-sample windows counts windows, not samples."""
    flat, offs = pack([[1, 2], [], (3,)], np.int32)
    assert flat.tolist() == [1, 2, 3] and offs.tolist() == [0, 2, 2, 3]
    flat, offs = pack([np.arange(4), np.arange(2)], np.float32, (2,))
    assert flat.shape == (3, 2) and offs.tolist() == [0, 2, 3]
