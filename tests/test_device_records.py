"""records.describe / layout of device arrays: objects exporting __cuda_array_interface__ (torch CUDA tensors, CuPy
arrays) are described by the same rules as numpy arrays -- row strides, views, the column-major hint, the dtypes -- with
the device flag and the producer stream on the descriptor.  Fake interface objects, so no GPU is needed."""
import numpy as np
import pytest

from mad_icp_b200 import records


class FakeDev:
    """a device array as far as the interface goes (its 'pointer' is the numpy buffer's address)"""

    def __init__(self, a, version=2, stream=None, strides=True):
        self._a = a
        cai = dict(shape=a.shape, typestr=a.dtype.str, data=(a.ctypes.data, False), version=version,
                   strides=tuple(a.strides) if strides else None)
        if version >= 3:
            cai["stream"] = stream
        self.__cuda_array_interface__ = cai


class Stream:
    def __init__(self, handle):
        self.cuda_stream = handle


def _same(a, dev):
    h, d = records.describe(a, 0.5, 80.0), records.describe(dev, 0.5, 80.0)
    for f in ("data", "n", "stride", "is_f32", "min_range", "max_range", "range_mode", "drop_nan"):
        assert getattr(h, f) == getattr(d, f), f
    assert list(h.offset) == list(d.offset)
    assert not h.on_device and h.stream is None and d.on_device
    return d


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_strides_and_views_match_numpy(dtype):
    base = np.zeros((100, 4), dtype)
    for a in (base, base[:, :3], base[1:, 1:4], base[::2, :3], np.zeros((100, 3), dtype), base[:1, :3]):
        _same(a, FakeDev(a))
    c = np.zeros((100, 3), dtype)
    d = _same(c, FakeDev(c, strides=False))  # C-contiguous: the interface may leave strides out
    assert d.stride == 3 * c.itemsize and list(d.offset) == [0, c.itemsize, 2 * c.itemsize]
    t = records.layout(FakeDev(base[:, :3]), 0.5, 80.0)
    assert len(t) == 13 and t[11] is True and t[12] == 0
    assert records.layout(base[:, :3])[11:] == (False, 0)


def test_column_major_is_rejected_with_the_hint():
    f = np.asfortranarray(np.zeros((100, 3), np.float32))
    with pytest.raises(ValueError, match="column-major"):
        records.describe(FakeDev(f))
    with pytest.raises(ValueError, match="column-major"):
        records.describe(FakeDev(np.zeros((3, 100), np.float32).T))


def test_dtypes_and_shapes_are_rejected():
    for a in (np.zeros((10, 3), np.int32), np.zeros((10, 3), np.float16), np.zeros((10, 3), ">f4"), np.zeros((10, 2), np.float32),
              np.zeros(10, np.float32), np.zeros((2, 10, 3), np.float32)):
        with pytest.raises(ValueError, match="device array"):
            records.describe(FakeDev(a))
    with pytest.raises(TypeError):
        records.describe([[0.0, 0.0, 0.0]])
    with pytest.raises(TypeError, match="host records"):
        records.range_mask(FakeDev(np.zeros((10, 3), np.float32)))


def test_stream_selection():
    a = np.zeros((10, 3), np.float32)
    assert records.describe(FakeDev(a)).stream == 0  # v2, not torch: the legacy default stream
    assert records.describe(FakeDev(a, version=3, stream=None)).stream == 0
    assert records.describe(FakeDev(a, version=3, stream=1234)).stream == 1234  # v3 entry
    assert records.describe(FakeDev(a, version=3, stream=1234), stream=77).stream == 77  # explicit int wins
    assert records.describe(FakeDev(a, version=3, stream=1234), stream=Stream(99)).stream == 99  # .cuda_stream
    assert records.describe(FakeDev(a), stream=Stream(5)).stream == 5
    assert records.layout(FakeDev(a, version=3, stream=42))[12] == 42
