"""A host replica of the Philox-4x32 generator behind every random stream of the kernels (csrc/common.cuh), and the
three streams built on it: the sampler's Gumbel uniforms (csrc/decode.cu), the forgetful causal mask
(csrc/tokens.cu) and the FFN dropout mask (csrc/ffn_mid.cu).

The replica is written from the published algorithm (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3",
SC'11): per round, with M0 = 0xD2511F53 and M1 = 0xCD9E8D57,
    (c0, c1, c2, c3) <- (hi(M1 c2) ^ c1 ^ k0,  lo(M1 c2),  hi(M0 c0) ^ c3 ^ k1,  lo(M0 c0)),
then the key is bumped by (0x9E3779B9, 0xBB67AE85).  The kernels use 7 rounds; the standard generator uses 10.
tests/test_sampling_gpu.py checks the kernels bit for bit against these mirrors."""
import numpy as np
import pytest

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32(c0, c1, c2, c3, k0, k1, rounds=7):
    """Philox-4x32-`rounds` of the counters (c0, c1, c2, c3) under the key (k0, k1): uint32 arrays (broadcast
    together) in, the four uint32 output words out."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & MASK32 for c in (c0, c1, c2, c3))
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(rounds):
        p0, p1 = M0 * c0, M1 * c2                      # < 2^64: exact in uint64
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & MASK32,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & MASK32)
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return tuple(w.astype(np.uint32) for w in (c0, c1, c2, c3))


def _key(seed):
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return seed & 0xFFFFFFFF, seed >> 32


def sampler_uniforms(seed, step, B, C):
    """float32 [B, C]: the uniform behind the Gumbel noise of class c in sequence b at sample index `step`
    (csrc/decode.cu sample_kernel): counter (c, b, step, 0x5a17), u = (x0 >> 8) / 2^24."""
    b, c = np.meshgrid(np.arange(B), np.arange(C), indexing="ij")
    x0 = philox4x32(c, b, step, 0x5A17, *_key(seed))[0]
    return ((x0 >> np.uint32(8)).astype(np.float64) / 2.0 ** 24).astype(np.float32)


def forgetful_keys(seed, stream_id, B, N):
    """uint32 [B, N]: the sort key of position p in row b (csrc/tokens.cu forgetful_mask_kernel): word x0 of counter
    (p, b, stream_lo, stream_hi), made odd; position 0 gets key 0 (never dropped)."""
    b, p = np.meshgrid(np.arange(B), np.arange(N), indexing="ij")
    sid = int(stream_id) & 0xFFFFFFFFFFFFFFFF
    x0 = philox4x32(p, b, sid & 0xFFFFFFFF, sid >> 32, *_key(seed))[0]
    keys = x0 | np.uint32(1)
    keys[:, 0] = 0
    return keys


def forgetful_mask(seed, stream_id, B, N, num_drop):
    """uint8 [B, N] keep mask: the num_drop largest keys of each row are dropped (equal keys: lower position first)."""
    keys = forgetful_keys(seed, stream_id, B, N)
    keep = np.ones((B, N), dtype=np.uint8)
    pos = np.arange(N)
    for b in range(B):
        order = np.lexsort((pos, -keys[b].astype(np.int64)))       # key descending, then position ascending
        keep[b, order[:num_drop]] = 0
    return keep


def dropout_keep(seed, layer, rows, Fp, drop_p):
    """bool [len(rows), Fp]: the FFN dropout keep flag of channel 8 j + i in chunk j (csrc/ffn_mid.cu dropout_keep8):
    counter (row_lo, row_hi, chunk, layer); 16-bit lane i (low half of word i // 2 first) kept iff
    lane >= uint32(drop_p * 65536.f) in fp32."""
    rows = np.asarray(rows, dtype=np.int64)
    r, ch = np.meshgrid(rows, np.arange(Fp // 8), indexing="ij")
    words = philox4x32(r & 0xFFFFFFFF, r >> 32, ch, layer, *_key(seed))
    lanes = np.stack([w for x in words for w in (x & np.uint32(0xFFFF), x >> np.uint32(16))], -1)   # [R, Fp/8, 8]
    thresh = np.uint32(np.float32(drop_p) * np.float32(65536.0))
    return (lanes >= thresh).reshape(len(rows), Fp)


# Known answers of at::Philox4_32 (ATen/core/PhiloxRNGEngine.h of the installed torch, whose engine takes the round
# count as an argument), printed by tools/philox_known_answers.cpp: (rounds, counter, key, output words).  The first
# three 10-round vectors are also the published Random123 known answers of philox4x32_10.
KNOWN_ANSWERS = [
    (10, (0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    (10, (0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    (10, (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
    (10, (0x00000007, 0x00000003, 0x0000000b, 0x00005a17), (0x9abcdef0, 0x12345678), (0x7ac3554a, 0x8f343625, 0x77592ff6, 0xe326bffd)),
    (10, (0x00000fff, 0x00000000, 0x0000015f, 0x00000002), (0x00003039, 0x00000000), (0x08c72084, 0xdc4d95c2, 0x96bf51ab, 0x57630f0b)),
    (7, (0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x5f6fb709, 0x0d893f64, 0x4f121f81, 0x4f730a48)),
    (7, (0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff), (0x5207ddc2, 0x45165e59, 0x4d8ee751, 0x8c52f662)),
    (7, (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0x4dfccaba, 0x190a87f0, 0xc47362ba, 0xb6b5242a)),
    (7, (0x00000007, 0x00000003, 0x0000000b, 0x00005a17), (0x9abcdef0, 0x12345678), (0x2ef502ca, 0xc4dae38a, 0xe0751171, 0x41ce3ac2)),
    (7, (0x00000fff, 0x00000000, 0x0000015f, 0x00000002), (0x00003039, 0x00000000), (0x3fa0cf95, 0xfe7e5fb7, 0xf204d0c2, 0x65bb6a8b)),
]


@pytest.mark.parametrize("rounds,ctr,key,out", KNOWN_ANSWERS, ids=[f"r{v[0]}-{i}" for i, v in enumerate(KNOWN_ANSWERS)])
def test_replica_matches_known_answers(rounds, ctr, key, out):
    got = philox4x32(*ctr, *key, rounds=rounds)
    assert tuple(int(w) for w in got) == out


def test_replica_is_vectorised_elementwise():
    """A batch of counters gives, element for element, the words of the scalar calls (broadcasting does not mix lanes)."""
    rng = np.random.default_rng(0)
    c = rng.integers(0, 2 ** 32, size=(4, 37), dtype=np.uint64)
    batch = philox4x32(c[0], c[1], c[2], c[3], 0xDEADBEEF, 0x01234567)
    for i in range(0, 37, 5):
        one = philox4x32(*(int(c[j, i]) for j in range(4)), 0xDEADBEEF, 0x01234567)
        assert tuple(int(w) for w in one) == tuple(int(w[i]) for w in batch)


def test_sampler_uniforms_are_24_bit_and_cover_the_unit_interval():
    u = sampler_uniforms(seed=3, step=0, B=64, C=1025)
    assert u.dtype == np.float32 and u.min() >= 0.0 and u.max() < 1.0
    assert np.array_equal(u * np.float32(2 ** 24), np.floor(u * np.float32(2 ** 24)))     # exact multiples of 2^-24
    assert abs(float(u.mean()) - 0.5) < 0.01 and abs(float(u.var()) - 1 / 12) < 0.005
    # every argument of the counter and both halves of the seed change the stream
    base = sampler_uniforms(seed=3, step=5, B=4, C=64)
    for other in (sampler_uniforms(seed=4, step=5, B=4, C=64), sampler_uniforms(seed=3 + (1 << 32), step=5, B=4, C=64),
                  sampler_uniforms(seed=3, step=6, B=4, C=64)):
        assert (other != base).mean() > 0.99
    assert (base[0] != base[1]).mean() > 0.99 and (base[:, :-1] != base[:, 1:]).mean() > 0.99


def test_forgetful_mirror_drops_exactly_num_drop_and_never_position_0():
    keep = forgetful_mask(seed=12345, stream_id=7, B=16, N=1024, num_drop=153)
    assert keep[:, 0].all() and ((keep == 0).sum(1) == 153).all()
    assert not np.array_equal(keep, forgetful_mask(seed=12345, stream_id=8, B=16, N=1024, num_drop=153))
    assert not np.array_equal(keep[0], keep[1])
    # num_drop = N - 1 drops everything but position 0
    assert forgetful_mask(seed=1, stream_id=2, B=2, N=50, num_drop=49).sum(1).tolist() == [1, 1]


@pytest.mark.parametrize("drop_p", [0.1, 0.5])
def test_dropout_mirror_keeps_one_minus_p(drop_p):
    keep = dropout_keep(seed=99, layer=3, rows=np.arange(512), Fp=1024, drop_p=drop_p)
    n = keep.size
    assert abs(1 - keep.mean() - drop_p) < 4 * np.sqrt(drop_p * (1 - drop_p) / n)
    # 16-bit lanes: the threshold of 0.1 is 6553 (6553.6 truncated), so P(drop) = 6553 / 65536
    thresh = int(np.float32(drop_p) * np.float32(65536.0))
    assert thresh == {0.1: 6553, 0.5: 32768}[drop_p]
    # rows beyond 2^32 use the high word of the row index
    lo = dropout_keep(seed=99, layer=3, rows=[5], Fp=128, drop_p=0.5)
    hi = dropout_keep(seed=99, layer=3, rows=[5 + (1 << 32)], Fp=128, drop_p=0.5)
    assert not np.array_equal(lo, hi)
