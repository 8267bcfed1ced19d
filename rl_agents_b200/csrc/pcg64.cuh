// numpy's PCG64 bit generator and the two Generator draws the reference
// planners consume, bit for bit (CPU twin + derivation: oracle/pcg64.py):
//   random_argmax -> np_random.choice(indices)   = integers(0, n)   (abstract.py:304-311)
//   rollout       -> np_random.choice(a, 1, p=p) = searchsorted(cdf, random(), 'right') (mcts.py:172)
#pragma once
#include <stdint.h>

namespace b2 {

struct Pcg64 {
    unsigned __int128 state, inc;
    uint32_t has_uint32, uinteger;

    __device__ __forceinline__ void load(const uint64_t* w) {
        state = ((unsigned __int128)w[0] << 64) | w[1];
        inc = ((unsigned __int128)w[2] << 64) | w[3];
        has_uint32 = (uint32_t)w[4];
        uinteger = (uint32_t)w[5];
    }
    __device__ __forceinline__ void store(uint64_t* w) const {
        w[0] = (uint64_t)(state >> 64);
        w[1] = (uint64_t)state;
        w[2] = (uint64_t)(inc >> 64);
        w[3] = (uint64_t)inc;
        w[4] = has_uint32;
        w[5] = uinteger;
    }
    __device__ __forceinline__ uint64_t next64() {
        const unsigned __int128 mult =
            ((unsigned __int128)0x2360ED051FC65DA4ULL << 64) | 0x4385DF649FCCF645ULL;
        state = state * mult + inc;
        const uint64_t hi = (uint64_t)(state >> 64), lo = (uint64_t)state;
        const uint64_t x = hi ^ lo;
        const unsigned rot = (unsigned)(hi >> 58);
        return (x >> rot) | (x << ((64 - rot) & 63));
    }
    __device__ __forceinline__ uint32_t next32() {
        if (has_uint32) {
            has_uint32 = 0;
            return uinteger;
        }
        const uint64_t n = next64();
        has_uint32 = 1;
        uinteger = (uint32_t)(n >> 32);
        return (uint32_t)n;
    }
    // The state after n calls of next32(), in O(log n): the buffered half first; then, for the m >= 1 halves left,
    // floor((m - 1) / 2) LCG steps (pcg_advance_lcg_128: square-and-multiply of next64's affine map) and the last
    // next64() as next32() runs it -- once when m is odd (its high half stays buffered), twice when m is even (the
    // buffered word, `uinteger`, then holds that step's high half, as after the last of the n calls).
    // CPU twin: tests/test_pcg64_skip.py::skip32.
    __device__ __forceinline__ void skip32(uint64_t n) {
        if (n == 0) return;
        if (has_uint32) {
            has_uint32 = 0;
            if (--n == 0) return;
        }
        unsigned __int128 cur_mult = ((unsigned __int128)0x2360ED051FC65DA4ULL << 64) | 0x4385DF649FCCF645ULL;
        unsigned __int128 cur_plus = inc, acc_mult = 1, acc_plus = 0;
        for (uint64_t delta = (n - 1) >> 1; delta > 0; delta >>= 1) {
            if (delta & 1) {
                acc_mult *= cur_mult;
                acc_plus = acc_plus * cur_mult + cur_plus;
            }
            cur_plus = (cur_mult + 1) * cur_plus;
            cur_mult *= cur_mult;
        }
        state = acc_mult * state + acc_plus;
        next32();
        if (!(n & 1)) next32();
    }
    __device__ __forceinline__ double random() { return (double)(next64() >> 11) * (1.0 / 9007199254740992.0); }
    // Generator.integers(0, n), 1 <= n < 2^32 (Lemire, buffered 32-bit halves)
    __device__ __forceinline__ uint32_t integers(uint32_t n) {
        const uint32_t rng = n - 1;
        if (rng == 0) return 0;
        const uint32_t rng_excl = rng + 1;
        uint64_t m = (uint64_t)next32() * rng_excl;
        uint32_t leftover = (uint32_t)m;
        if (leftover < rng_excl) {
            const uint32_t threshold = (0xFFFFFFFFu - rng) % rng_excl;
            while (leftover < threshold) {
                m = (uint64_t)next32() * rng_excl;
                leftover = (uint32_t)m;
            }
        }
        return (uint32_t)(m >> 32);
    }
    // np.random.default_rng(seed) for a seed below 2^32 (an env's `seed(np_random.randint(2**30))`): the words of
    // SeedSequence(seed).generate_state(4, uint64) -- one entropy word, pool size 4 -- then pcg64_set_seed
    // (state 0, inc = initseq << 1 | 1, step, state += initstate, step).  CPU twin: oracle/seed_sequence.py.
    __device__ __forceinline__ void seed_from(uint32_t seed) {
        uint32_t hash_const = 0x43B0D7E5u;
        auto hashmix = [&hash_const](uint32_t v) {
            v ^= hash_const;
            hash_const *= 0x931E8875u;
            v *= hash_const;
            return v ^ (v >> 16);
        };
        auto mix = [](uint32_t x, uint32_t y) {
            const uint32_t r = 0xCA01F9DDu * x - 0x4973F715u * y;
            return r ^ (r >> 16);
        };
        uint32_t pool[4];
        pool[0] = hashmix(seed);
#pragma unroll
        for (int i = 1; i < 4; ++i) pool[i] = hashmix(0u);
#pragma unroll
        for (int src = 0; src < 4; ++src)
#pragma unroll
            for (int dst = 0; dst < 4; ++dst)
                if (src != dst) pool[dst] = mix(pool[dst], hashmix(pool[src]));
        uint32_t hb = 0x8B51F9DDu, w[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t v = pool[i & 3] ^ hb;
            hb *= 0x58F38DEDu;
            v *= hb;
            w[i] = v ^ (v >> 16);
        }
        const unsigned __int128 initstate = ((unsigned __int128)(((uint64_t)w[1] << 32) | w[0]) << 64) |
                                            (((uint64_t)w[3] << 32) | w[2]);
        const unsigned __int128 initseq = ((unsigned __int128)(((uint64_t)w[5] << 32) | w[4]) << 64) |
                                          (((uint64_t)w[7] << 32) | w[6]);
        state = 0;
        inc = (initseq << 1) | 1u;
        next64();
        state += initstate;
        next64();
        has_uint32 = 0;
        uinteger = 0;
    }
};

}  // namespace b2
