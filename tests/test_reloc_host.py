"""The keyframe database's rules without a GPU: the numpy restatement (tests/reloc_walk.py) of the splitmix64 fern
tables, the colour block means, nibble packing and distances, the query order and the add rule."""
import numpy as np
import pytest

from tests import reloc_walk as W


def test_splitmix64_matches_the_published_sequence():
    # the first outputs of splitmix64 from state 0 (Steele, Lea and Flood's reference sequence)
    state, out = 0, []
    for _ in range(4):
        state, v = W.splitmix64(state)
        out.append(v)
    assert out == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F, 0xF88BB8A8724C81EC]


def test_fern_tables_take_six_draws_per_fern_in_order():
    t = W.fern_tables(8, 0, 80, 60, 0.3, 4.0)
    # fern 0: x, y, r, g from the four values above, then b and the depth threshold from draws 5 and 6
    assert t["x"][0] == (0xE220A8397B1DCDAF >> 32) % 80 == 0xE220A839 % 80
    assert t["y"][0] == 0x6E789E6A % 60
    assert t["r"][0] == 0x06 and t["g"][0] == 0xF8
    state = 0
    values = []
    for _ in range(12):
        state, v = W.splitmix64(state)
        values.append(v)
    assert t["b"][0] == values[4] >> 56
    lo, hi = float(np.float32(0.3)), float(np.float32(4.0))
    assert t["depth"][0] == lo + (hi - lo) * ((values[5] >> 11) * 2.0 ** -53)
    assert t["x"][1] == (values[6] >> 32) % 80 and t["y"][1] == (values[7] >> 32) % 60
    assert ((t["depth"] >= lo) & (t["depth"] < hi)).all()


@pytest.mark.parametrize("size,level", [((641, 479), 3), ((101, 77), 2), ((640, 480), 4), ((33, 31), 1)])
def test_colour_block_means_at_odd_sizes(size, level):
    W_, H_ = size
    rng = np.random.default_rng(W_ * H_)
    color = rng.integers(0, 256, (H_, W_, 3), dtype=np.uint8)
    w, h = W.fern_size(W_, level), W.fern_size(H_, level)
    got = W.block_means(color, w, h)
    for y in range(0, h, max(1, h // 7)):
        for x in range(0, w, max(1, w // 7)):
            block = color[H_ * y // h:H_ * (y + 1) // h, W_ * x // w:W_ * (x + 1) // w].reshape(-1, 3).astype(np.int64)
            n = block.shape[0]
            assert n > 0
            assert (got[y, x] == (block.sum(0) + n // 2) // n).all(), (x, y)
    # a block of 2 pixels rounds half up: (1 + 2 + 1) // 2 = 2
    two = np.array([[[1, 1, 1], [2, 2, 2]]], np.uint8)
    assert (W.block_means(two, 1, 1) == 2).all()


def test_nibble_packing_and_distance_on_hand_built_codes():
    nibbles = np.arange(16, dtype=np.uint32) % 16
    code = W.pack(nibbles)
    assert code.tolist() == [0x76543210, 0xFEDCBA98]
    assert (W.unpack(code) == nibbles).all()
    other = nibbles.copy()
    other[[0, 5, 9]] ^= np.array([8, 1, 15], np.uint32)   # three ferns differ, by one, one and four bits
    assert W.distance(code, W.pack(other)) == 3
    assert W.distance(code, code) == 0
    assert W.distance(W.pack(np.zeros(16, np.uint32)), W.pack(np.full(16, 15, np.uint32))) == 16


def test_query_orders_ties_by_index_and_applies_the_bound():
    ferns = 16
    base = np.zeros(ferns, np.uint32)
    def at(k):
        n = base.copy()
        n[:k] = 1
        return W.pack(n)
    codes = [at(4), at(2), at(4), at(1), at(2), at(9)]
    idx, dist = W.query(W.pack(base), codes, 8, 0.5, ferns)
    assert idx.tolist() == [3, 1, 4, 0, 2] and dist.tolist() == [1, 2, 2, 4, 4]   # 9 > 0.5 * 16 is dropped
    idx, _ = W.query(W.pack(base), codes, 3, 1.0, ferns)
    assert idx.tolist() == [3, 1, 4]
    idx, _ = W.query(W.pack(base), [], 3, 1.0, ferns)
    assert idx.size == 0


def test_add_rule_at_the_threshold_at_capacity_and_with_force():
    ferns = 16
    db = W.Database(ferns, capacity=3, add_fraction=0.25)   # bound 4.0: a distance of 4 is not new, 5 is
    zero = np.zeros(ferns, np.uint32)
    def code(k):
        n = zero.copy()
        n[:k] = 2
        return W.pack(n)
    I = np.eye(4, dtype=np.float32)[:3]
    assert db.add(code(0), I) == (0, False)          # empty database
    assert db.add(code(4), I) == (-1, False)         # at the bound
    assert db.add(code(5), I) == (1, False)          # beyond it
    assert db.add(code(0), I, force=True) == (2, False)
    assert db.add(code(16), I) == (-1, True)         # new, but the database is full
    assert db.add(code(0), I) == (-1, False)         # not new: full is not reported
    assert db.add(code(0), I, force=True) == (-1, True)
    assert len(db.codes) == 3


def test_encode_restatement_on_a_hand_built_frame():
    enc = W.Encoder(64, 48, level=2, ferns=16, seed=7, min_depth=0.5, max_depth=2.0)
    depth = np.full((48, 64), 5000, np.uint16)                    # 1 m everywhere
    color = np.zeros((48, 64, 3), np.uint8)
    color[..., 0] = 255
    nib = enc.nibbles(depth, color)
    t = enc.tables
    assert ((nib & 1) == 1).all()                                 # R = 255 >= any threshold
    assert ((nib >> 1 & 1) == (t["g"] == 0)).all() and ((nib >> 2 & 1) == (t["b"] == 0)).all()
    assert ((nib >> 3 & 1) == (5000.0 >= t["depth"] * 5000.0)).all()
    assert ((enc.nibbles(np.zeros_like(depth), color) >> 3) == 0).all()   # D = 0 never sets bit 3
