"""CPU: tests/grid_ref.py, the restatement fg_image_grid is held to, on hand-computed sheets: values on and one ulp
either side of k/255, a constant grid, a ragged last row filled with the maximum, padding with nrow > count, one
channel, NaN, and the ordered keys of the exact minimum / maximum."""
import numpy as np

import grid_ref as G


def test_k_over_255_and_one_ulp_either_side():
    """min 0 and max 1 make minmax the identity; fl(k/255) * 255 is exactly k in float32, the float below it gives
    k - 1 after truncation, the float above it k."""
    vals, want = [np.float32(0), np.float32(1)], [0, 255]
    for k in range(1, 255):
        x = np.float32(k / 255)
        vals += [np.nextafter(x, np.float32(0)), x, np.nextafter(x, np.float32(2))]
        want += [k - 1, k, k]
    img = np.array(vals, np.float32).reshape(1, 1, 1, -1)
    got = G.grid(img, nrow=1)
    assert got.shape == (1, 1, len(vals))
    np.testing.assert_array_equal(got[0, 0], np.array(want, np.uint8))


def test_min_max_are_shifted_and_scaled():
    """[-1, 0, 3]: shifted by 1, divided by 4 -> 0, 0.25, 1 -> 0, 63 (63.75 truncated), 255."""
    img = np.array([-1, 0, 3], np.float32).reshape(1, 1, 1, 3)
    np.testing.assert_array_equal(G.grid(img, 1)[0, 0], [0, 63, 255])


def test_constant_grid_is_shifted_not_scaled():
    img = np.full((4, 3, 2, 2), 0.7, np.float32)
    got = G.grid(img, nrow=2, padding=2)
    assert got.shape == (3, 2 * 4, 2 * 4)
    assert (got == 0).all()


def test_ragged_last_row_fill_becomes_255():
    """5 images, 2 per row: 3 rows, the last cell is the fill (the maximum), 255 after minmax."""
    img = np.stack([np.full((3, 2, 3), v, np.float32) for v in (0.2, 0.3, 0.4, 0.5, 0.6)])
    got = G.grid(img, nrow=2)
    assert got.shape == (3, 6, 6)
    # (v - 0.2) / 0.4 in float32, * 255, truncated
    expect = {0: 0, 1: 63, 2: 127, 3: 191, 4: 255}
    for k, b in expect.items():
        y, x = divmod(k, 2)
        assert (got[:, 2 * y:2 * y + 2, 3 * x:3 * x + 3] == b).all(), (k, b)
    assert (got[:, 4:6, 3:6] == 255).all()


def test_padding_nrow_above_count_one_channel():
    """3 gray 2x2 images, nrow 8: one row of three 4x4 cells, the image at offset 1, the border the fill."""
    img = np.stack([np.array([[0, 1], [2, 3]], np.float32) + 4 * k for k in range(3)])[:, None]
    got = G.grid(img, nrow=8, padding=2)
    assert got.shape == (1, 4, 12)
    want = np.full((4, 12), 255, np.uint8)
    for k in range(3):
        # (v - 0) / 11 * 255 truncated
        want[1:3, 4 * k + 1:4 * k + 3] = [[int(np.float32(np.float32(v / np.float32(11)) * np.float32(255)))
                                           for v in row] for row in img[k, 0].astype(np.float32)]
    np.testing.assert_array_equal(got[0], want)
    assert want[1, 1] == 0 and want[2, 10] == 255 and want[1, 2] == 23  # 1/11 * 255 = 23.18


def test_order_selects_and_orders():
    img = np.stack([np.full((1, 1, 1), v, np.float32) for v in (5, 1, 3, 9)])
    got = G.grid(img, nrow=4, order=[3, 1, 2])
    np.testing.assert_array_equal(got[0, 0], [255, 0, 63])  # 9, 1, 3: (v - 1) / 8 * 255 = 255, 0, 63.75


def test_nan_is_left_out_and_gives_zero():
    img = np.array([0.5, np.nan, 1.5, 1.0], np.float32).reshape(1, 1, 1, 4)
    np.testing.assert_array_equal(G.grid(img, 1)[0, 0], [0, 0, 255, 127])
    assert G.extremes(np.full(3, np.nan, np.float32)) == (0, 0)


def test_ordered_keys_and_signed_zero():
    x = np.array([-np.inf, -2.5, -0.0, 0.0, 1e-45, 3.0, np.inf], np.float32)
    k = G.ordered_keys(x)
    assert (np.diff(k.astype(np.int64)) > 0).all()
    for v, kk in zip(x, k):
        assert G.key_value(kk).tobytes() == v.tobytes()
