"""numpy's PCG64 stream, followed in Python ints, so fit() can draw its initial factors on the device.

``Generator.random(size, dtype=np.float32)`` takes one 32-bit half of a 64-bit PCG64 draw per value: the low half of a
new draw first, the high half buffered (``has_uint32`` / ``uinteger`` of the state dict) for the next value, across
calls too.  A 64-bit draw steps the 128-bit LCG state first, s = s * MULT + inc (mod 2^128), then outputs
rotr64(hi ^ lo, hi >> 58) of the new state.  The device fill (als_factors_fill_pcg64) computes the same values in
parallel; these functions give it the state to start from and give the generator the state numpy would leave.
"""
import numpy as np

MULT = 0x2360ED051FC65DA44385DF649FCCF645
MASK128 = (1 << 128) - 1
MASK64 = (1 << 64) - 1


def device_drawable(gen):
    """True when gen's draws can be reproduced on the device: its bit generator is exactly numpy's PCG64 (the one
    default_rng and check_random_state build); PCG64DXSM, Philox, MT19937 and SFC64 are drawn on the host."""
    return type(gen.bit_generator) is np.random.PCG64


def get_state(gen):
    """(state, inc, has_uint32, uinteger) of a PCG64 Generator, as Python ints."""
    st = gen.bit_generator.state
    return st["state"]["state"], st["state"]["inc"], st["has_uint32"], st["uinteger"]


def set_state(gen, state):
    """Writes (state, inc, has_uint32, uinteger) back into gen.  (bit_generator.advance() would clear has_uint32.)"""
    s, inc, has, u = state
    gen.bit_generator.state = {"bit_generator": "PCG64", "state": {"state": s, "inc": inc},
                               "has_uint32": has, "uinteger": u}


def advance(s, inc, k):
    """The LCG state k steps after s (Brown's jump-ahead: O(log k) 128-bit multiply-adds)."""
    acc_mult, acc_plus, mult, plus = 1, 0, MULT, inc
    while k > 0:
        if k & 1:
            acc_mult = acc_mult * mult & MASK128
            acc_plus = (acc_plus * mult + plus) & MASK128
        plus = (mult + 1) * plus & MASK128
        mult = mult * mult & MASK128
        k >>= 1
    return (acc_mult * s + acc_plus) & MASK128


def output(s):
    """The 64-bit output of a draw whose stepped state is s (XSL-RR)."""
    hi, lo = s >> 64, s & MASK64
    rot = hi >> 58
    x = hi ^ lo
    return ((x >> rot) | (x << (64 - rot))) & MASK64


def after_float32_draws(state, n):
    """The (state, inc, has_uint32, uinteger) numpy leaves after n values of random(..., dtype=np.float32) from state."""
    s, inc, has, u = state
    if n == 0:
        return state
    m = n - has  # values taken from new 64-bit draws
    steps = (m + 1) // 2
    if steps:
        s = advance(s, inc, steps)
        u = output(s) >> 32
    return s, inc, m % 2, u


def generator_at(state):
    """A new PCG64 Generator in the given (state, inc, has_uint32, uinteger)."""
    gen = np.random.Generator(np.random.PCG64())
    set_state(gen, state)
    return gen
