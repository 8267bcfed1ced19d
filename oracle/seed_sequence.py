"""Pure-Python restatement of how `np.random.default_rng(seed)` seeds its PCG64 -- TEST INFRASTRUCTURE.

The sampled env of sparse sampling is re-seeded before every step (`seed(np_random.randint(2**30))`, then
`default_rng(seed)`), so the device replays this seeding for every sample.  For a seed below 2**32 it is
SeedSequence(seed).generate_state(4, np.uint64) -- one entropy word, pool size 4, `hashmix` / `mix` -- followed by
pcg64_set_seed (pcg_setseq_128_srandom_r: state 0, inc = initseq << 1 | 1, step, state += initstate, step).
Algorithm source: numpy/random/bit_generator.pyx and numpy/random/src/pcg64/pcg64.h; pinned against numpy itself
(tests/test_sparse_sampling_oracle.py).  The CUDA twin is Pcg64::seed_from in rl_agents_b200/csrc/pcg64.cuh.
"""
from oracle.pcg64 import MASK128, PCG64

SS_INIT_A, SS_MULT_A = 0x43B0D7E5, 0x931E8875
SS_INIT_B, SS_MULT_B = 0x8B51F9DD, 0x58F38DED
SS_MIX_MULT_L, SS_MIX_MULT_R = 0xCA01F9DD, 0x4973F715
MASK32 = 0xFFFFFFFF


def seed_sequence_state(seed):
    """SeedSequence(seed).generate_state(4, np.uint64) for 0 <= seed < 2**32."""
    seed = int(seed)
    assert 0 <= seed <= MASK32
    hash_const = [SS_INIT_A]

    def hashmix(value):
        value = (value ^ hash_const[0]) & MASK32
        hash_const[0] = (hash_const[0] * SS_MULT_A) & MASK32
        value = (value * hash_const[0]) & MASK32
        return value ^ (value >> 16)

    def mix(x, y):
        r = (SS_MIX_MULT_L * x - SS_MIX_MULT_R * y) & MASK32
        return r ^ (r >> 16)

    pool = [hashmix(seed), hashmix(0), hashmix(0), hashmix(0)]
    for i_src in range(4):
        for i_dst in range(4):
            if i_src != i_dst:
                pool[i_dst] = mix(pool[i_dst], hashmix(pool[i_src]))
    hb, words = SS_INIT_B, []
    for i in range(8):
        v = pool[i % 4] ^ hb
        hb = (hb * SS_MULT_B) & MASK32
        v = (v * hb) & MASK32
        words.append(v ^ (v >> 16))
    return [words[2 * i] | (words[2 * i + 1] << 32) for i in range(4)]


def pcg64_from_seed(seed):
    """The bit generator of np.random.default_rng(seed), 0 <= seed < 2**32: pcg64_set_seed with
    initstate = w0:w1, initseq = w2:w3 of seed_sequence_state."""
    w = seed_sequence_state(seed)
    initstate, initseq = (w[0] << 64) | w[1], (w[2] << 64) | w[3]
    g = PCG64(0, ((initseq << 1) | 1) & MASK128)
    g.next64()
    g.state = (g.state + initstate) & MASK128
    g.next64()
    return g
