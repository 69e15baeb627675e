"""The host Philox4x32-10 (oracle/philox.py) against known answers, so that the sampling-kernel tests can predict
every uniform the kernel draws.

* the Random123 known-answer vectors of philox4x32 with 10 rounds;
* words and uniforms of curand's own ``curand_init(seed, 0, offset)`` / ``curand`` / ``curand_uniform``, recorded
  from the CUDA 12.9 header compiled for the host, at seeds 0, 1234 and 2^63 - 1 and offsets that are and are not
  multiples of 4 (one beyond 2^32 blocks, so the counter's high word carries);
* the ends of ``curand_uniform``'s range and the kernel's offset advance."""
import numpy as np
import pytest

from oracle import philox as P


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_random123_known_answers(ctr, key, want):
    assert P.philox4x32_10(np.array(ctr, dtype=np.uint32), key).tolist() == list(want)


CURAND = [   # seed, offset, the first 6 words of curand(), the first 6 curand_uniform() values (printed with %.9g)
    (0, 0, [1713891541, 3781805453, 3159862348, 2600524760, 4175744164, 1555169499],
     [0.399046481, 0.880520225, 0.735712767, 0.605481863, 0.972241223, 0.362091124]),
    (0, 5, [1555169499, 2980410603, 159317863, 83534633, 1372009126, 605361069],
     [0.362091124, 0.693930924, 0.037094079, 0.0194494221, 0.319445759, 0.140946612]),
    (0, 0xfffffffffff, [460058700, 825917295, 2545093161, 1363227784, 195859037, 358347136],
     [0.10711576, 0.192298859, 0.592575669, 0.317401201, 0.0456019863, 0.0834341943]),
    (1234, 0, [546353992, 3665621163, 1140953199, 3419031310, 2666454581, 482218876],
     [0.12720795, 0.853468955, 0.265648872, 0.796055257, 0.620832324, 0.112275332]),
    (1234, 5, [482218876, 4196888723, 343858512, 1070188760, 4228315704, 3424062247],
     [0.112275332, 0.977164328, 0.0800607949, 0.249172732, 0.984481454, 0.797226608]),
    (1234, 0xfffffffffff, [4198382586, 3288568338, 2475882233, 1061194149, 3135560696, 1680073161],
     [0.977512121, 0.765679479, 0.576461256, 0.247078523, 0.730054617, 0.391172528]),
    (2 ** 63 - 1, 0, [854020009, 2481712373, 4176245556, 227446781, 137484036, 3309058435],
     [0.198842034, 0.577818692, 0.972357929, 0.0529565811, 0.0320104957, 0.770450234]),
    (2 ** 63 - 1, 5, [3309058435, 3372859969, 2360952418, 2504880811, 2707673398, 2132043920],
     [0.770450234, 0.785305142, 0.549702048, 0.583213031, 0.630429327, 0.496405154]),
    (2 ** 63 - 1, 0xfffffffffff, [3868320289, 4010490648, 3967804083, 476067277, 132539497, 595186739],
     [0.900663495, 0.933765113, 0.923826396, 0.110843047, 0.0308592562, 0.138577715]),
]


@pytest.mark.parametrize("seed,offset,w,u", CURAND)
def test_stream_matches_curand(seed, offset, w, u):
    assert P.words(seed, offset, 6).tolist() == w
    got = P.uniforms(seed, offset, 6)
    assert got.dtype == np.float32
    assert ["%.9g" % x for x in got] == ["%.9g" % x for x in u]        # %.9g round-trips fp32: bit for bit


def test_offsets_are_word_indices_of_one_stream():
    seed = 99
    base = P.words(seed, 0, 64)
    offs = np.arange(40, dtype=np.uint64)
    win = P.words(seed, offs, 8)                                       # vectorised over offsets
    for o in offs:
        assert win[o].tolist() == base[o:o + 8].tolist()
    assert len(set(base.tolist())) == 64


def test_uniform_range_and_advance():
    u = P.to_uniform(np.array([0, 1, 0xffffff7f, 0xffffffff], dtype=np.uint32))
    assert u[0] == np.float32(2.0 ** -33) and u[1] == np.float32(2.0 ** -33 + 2.0 ** -32)
    assert u[3] == np.float32(1.0)                                     # (0, 1]: 1 is reachable, 0 is not
    assert 0 < u[2] <= 1
    assert [P.advance(n) for n in (0, 1, 3, 4, 5, 8, 9)] == [0, 4, 4, 4, 8, 8, 12]
