"""rsem_b200_mt19937_jump on the host (no GPU): the boost::mt19937 state after J draws, checked against numpy's MT19937
walked draw by draw.  numpy's state (key, pos) is boost's (words, index): pos == 624 means "twist before the next
draw".  The jump lengths are those rsem-simulate-reads uses over several devices: the start g W of device g's first
window, and (G - 1) W - L between a device's windows, at the default window W = 2^22."""
import numpy as np
import pytest

W = 1 << 22
L = 2 * (6 + 2 * (2 * 50 + 1)) + 8  # the simulator's L for paired-end 2 x 50 bases: the longest attempt, in words
SEEDS = [0, 1, 7, 2**32 - 1]


@pytest.fixture(scope="module")
def lib(built):
    import rsem_b200
    return rsem_b200.load_library()


def boost_seed(seed):
    """boost::mt19937(seed): the words, then index 624"""
    x = [seed & 0xFFFFFFFF]
    for i in range(1, 624):
        x.append((1812433253 * (x[-1] ^ (x[-1] >> 30)) + i) & 0xFFFFFFFF)
    return np.array(x + [624], np.uint32)


def walk(state, J):
    """the state after J draws, one draw at a time (numpy's MT19937)"""
    bg = np.random.MT19937()
    bg.state = {"bit_generator": "MT19937", "state": {"key": state[:624].copy(), "pos": int(state[624])}}
    while J > 0:
        step = min(J, 1 << 24)
        bg.random_raw(step)
        J -= step
    st = bg.state["state"]
    return np.concatenate([st["key"].astype(np.uint32), [np.uint32(st["pos"])]])


def draws(state, n):
    bg = np.random.MT19937()
    bg.state = {"bit_generator": "MT19937", "state": {"key": state[:624].copy(), "pos": int(state[624])}}
    return bg.random_raw(n)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("J", [0, 1, 396, 397, 623, 624, 625, 1247, 1248, W - L])
def test_jump_equals_walk(lib, seed, J):
    s = boost_seed(seed)
    got = lib.mt19937_jump(s, J)
    assert np.array_equal(got, walk(s, J))


@pytest.mark.parametrize("G", range(2, 9))
def test_jump_between_windows(lib, G):
    """a device's jump from the end of window w (W + L words on) to the start of window w + G"""
    s = lib.mt19937_jump(boost_seed(7), W + L)
    J = (G - 1) * W - L
    assert np.array_equal(lib.mt19937_jump(s, J), walk(s, J))


@pytest.mark.parametrize("G", [2, 3])
def test_first_window_starts(lib, G):
    """device g starts at word g W of the stream: the jumped state draws what the walk draws there"""
    s = boost_seed(11)
    stream = draws(s, G * W + 5)
    for g in range(G):
        assert np.array_equal(draws(lib.mt19937_jump(s, g * W), 5), stream[g * W:g * W + 5])


@pytest.mark.parametrize("idx", [0, 1, 623, 624])
@pytest.mark.parametrize("J", [0, 1, 623, 624, 625, 20000, 3 * W])
def test_index_word(lib, idx, J):
    """any index the state can hold, including 0 (the words not yet drawn from) and 624 (twist first)"""
    s = walk(boost_seed(1), 5000)
    s[624] = idx
    assert np.array_equal(lib.mt19937_jump(s, J), walk(s, J))


@pytest.mark.parametrize("J1,J2", [(2**35, 3), (2**34 + 17, 2**34 - 14), (12345, 2**35 - 12342), (W - L, W * 7 + 1)])
def test_jumps_compose(lib, J1, J2):
    """offsets too long to walk: one jump of J1 + J2 equals J1 then J2"""
    s = boost_seed(1)
    one = lib.mt19937_jump(s, J1 + J2)
    assert np.array_equal(one, lib.mt19937_jump(lib.mt19937_jump(s, J1), J2))
    assert int(one[624]) == (int(s[624]) + J1 + J2 - 1) % 624 + 1


def test_long_jump_equals_walk(lib):
    s = boost_seed(2**32 - 1)
    J = 7 * W + 2**24 + 5
    assert np.array_equal(lib.mt19937_jump(s, J), walk(s, J))


def test_rejects_bad_index(lib):
    import rsem_b200
    s = boost_seed(1)
    s[624] = 625
    with pytest.raises(rsem_b200.RsemB200Error, match="index"):
        lib.mt19937_jump(s, 1)
