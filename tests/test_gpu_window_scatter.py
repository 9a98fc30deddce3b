"""The window-scatter phase D2 (k_distribute_window, W % 4 == 0) on shapes whose tile edges fall
inside the image in both directions: partial tiles at the right and bottom borders, windows
clamped at every image edge, batched layout."""
import pytest

from test_gpu_parity import test_batched_and_odd_shapes_vs_oracle as _shape_vs_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("b,f,h,w", [(2, 3, 40, 100), (1, 2, 72, 136)])
def test_partial_window_tiles_vs_oracle(b, f, h, w):
    _shape_vs_oracle(b, f, h, w)
