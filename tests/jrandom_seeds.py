"""Seeds that force java.util.Random's nextInt(bound) rejection loop at a chosen draw.

nextInt(bound) with a bound that is not a power of two rejects a raw next(31) value u when
u - u % bound + bound - 1 >= 2^31 (int overflow in Java) and draws again, so every later pick of the execution moves by
one draw.  At this project's bounds that happens about once in 10^9 draws, so no ordinary seed range reaches it.

The generator's state after k steps is s_k = (s_{k-1} * 0x5DEECE66D + 0xB) mod 2^48, and next(31) is its top 31 bits.
The multiplier is odd, hence invertible mod 2^48: seed_for runs the LCG back from a chosen s_k to the seed.  One
execution can have only one forced draw, since a second would need 62 bits of a 48-bit state; low17 picks one of 2^17
seeds with the same forced value."""

MULT, ADD, MASK = 0x5DEECE66D, 0xB, (1 << 48) - 1
INV = pow(MULT, -1, 1 << 48)
TOP = 1 << 31

# the largest raw value: rejected by every bound that is not a power of two
ALWAYS = TOP - 1


def seed_for(k, top31, low17=0):
    """A Java long seed whose k-th next(31) (k >= 1) is top31.  The same state fixes next(26) (top31 >> 5) and
    next(27) (top31 >> 4): the first and second halves of a nextDouble that starts at draw k."""
    assert k >= 1 and 0 <= top31 < TOP and 0 <= low17 < (1 << 17)
    s = (top31 << 17) | low17
    for _ in range(k):
        s = ((s - ADD) * INV) & MASK
    return s ^ MULT


def rejects(u, n):
    """Java's rejection test of raw value u under nextInt(n)."""
    if n & (n - 1) == 0:
        return False
    return u - u % n + n - 1 >= TOP


def raw_draws(seed, k):
    """The first k raw next(31) values of new Random(seed)."""
    s = (seed ^ MULT) & MASK
    out = []
    for _ in range(k):
        s = (s * MULT + ADD) & MASK
        out.append(s >> 17)
    return out


def crafted(positions, raw=ALWAYS, per_position=4):
    """{position: [seeds]}: per_position seeds per position whose draw at that position is `raw`."""
    return {k: [seed_for(k, raw, 0x1000 * j + 0x5A5 + k) for j in range(per_position)] for k in positions}
