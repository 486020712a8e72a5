"""CPU: the algebra of the tensor-core operand tiles (covins_b200/csrc/tc_match.cu, namespace xt), restated in numpy.

The matching kernel never computes a Hamming distance explicitly: query bytes 0/2 (u8) against train bytes 0/-128 (s8) plus one
32-byte key slice on each side make the s32 accumulator equal to  Hamming << 7 | row-in-tile.  This test pins the encoding rules
(byte values, the decomposition of popc(t) / 2 popc(q) into bytes that fit s8 / u8, the sentinel of rows past a keyframe's end)
and the bounds the packed 16-bit epilogue relies on."""
import numpy as np


def _bits(rows):                      # [n, 32] u8 → [n, 256] 0/1
    return np.unpackbits(rows, axis=1, bitorder="little").astype(np.int64)


def _query_operand(q):                # per query row: 256 data bytes (0/2, u8) + key slice [1,128,128,128,c4,c5,c6,0...]
    b = _bits(q)
    pq = b.sum(1)
    c4 = np.minimum(2 * pq, 255); c5 = np.minimum(2 * pq - c4, 255); c6 = 2 * pq - c4 - c5
    key = np.zeros((len(q), 32), np.int64)
    key[:, 0] = 1; key[:, 1:4] = 128; key[:, 4] = c4; key[:, 5] = c5; key[:, 6] = c6
    a = np.concatenate([2 * b, key], 1)
    assert a.min() >= 0 and a.max() <= 255                       # u8
    return a


def _train_operand(t, n_valid):       # per tile row: 256 data bytes (0/-128, s8) + key slice [col,p1,p2,p3,64,64,64,0...]
    b = _bits(t)
    pt = b.sum(1)
    p1 = np.minimum(pt, 127); p2 = np.minimum(pt - p1, 127); p3 = pt - p1 - p2
    key = np.zeros((len(t), 32), np.int64)
    key[:, 0] = np.arange(len(t)); key[:, 1] = p1; key[:, 2] = p2; key[:, 3] = p3; key[:, 4:7] = 64
    data = -128 * b
    inv = np.arange(len(t)) >= n_valid                           # rows past the keyframe's end: no data, key bytes 127 x 4
    data[inv] = 0; key[inv] = 0; key[inv, 0:4] = 127
    o = np.concatenate([data, key], 1)
    assert o.min() >= -128 and o.max() <= 127                    # s8
    return o


def test_accumulator_is_the_packed_sort_key():
    rng = np.random.default_rng(0)
    q = rng.integers(0, 256, (128, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (128, 32), dtype=np.uint8)
    # extremes: all-zero / all-one descriptors on both sides (popc 0 and 256, Hamming 0 and 256)
    q[0] = 0; q[1] = 255; t[0] = 0; t[1] = 255; t[2] = q[5]
    n_valid = 104                                                # the last tile of a 1000-row keyframe
    acc = _query_operand(q) @ _train_operand(t, n_valid).T       # s32 GEMM, K = 288
    ham = (_bits(q)[:, None, :] != _bits(t)[None, :, :]).sum(2)
    col = np.arange(128)[None, :]
    assert np.array_equal(acc[:, :n_valid], (ham[:, :n_valid] << 7) | col[:, :n_valid])
    assert acc[:, :n_valid].max() <= 32895 < 32896               # kKeyInvalid: every real key is below it
    assert np.all(acc[:, n_valid:] == 127 + 3 * 127 * 128)       # 48895: rows past the end never enter a list
    assert acc.min() >= 0 and acc.max() < 65536                  # packing two columns into one 32-bit register loses nothing
    assert ham[5, 2] == 0 and acc[5, 2] == 2                     # a perfect match: key = column only


def test_key_order_is_distance_then_row():
    """ascending key order within a tile = (distance, row index): the order OpenCV's knnMatch keeps for ties"""
    rng = np.random.default_rng(1)
    q = rng.integers(0, 256, (4, 32), dtype=np.uint8)
    base = rng.integers(0, 256, (8, 32), dtype=np.uint8)
    t = base[rng.integers(0, 8, 128)]                            # many exact duplicates → ties
    acc = _query_operand(q) @ _train_operand(t, 128).T
    ham = (_bits(q)[:, None, :] != _bits(t)[None, :, :]).sum(2)
    for r in range(4):
        order = np.argsort(acc[r], kind="stable")
        ref = np.lexsort((np.arange(128), ham[r]))
        assert np.array_equal(order, ref)
