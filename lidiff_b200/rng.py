"""numpy's legacy `randn` and torch's CPU `randperm` drawn on the GPU, bit for bit, leaving the host generators where the host calls
would leave them.

    r = numpy_randn(1, n, 3, device="cuda")         # == torch.from_numpy(np.random.randn(1, n, 3)), and np.random's state after it
    p = torch_randperm(n, device="cuda")            # == torch.randperm(n), and torch's CPU generator state after it

Both read the host generator's MT19937 state, draw its word stream on the device (lb2_mt19937_words) and write the state after the
consumed words back.  numpy_randn runs numpy's polar method (lb2_legacy_gauss, with glibc's log: DESIGN.md §3, device random draws);
torch_randperm runs torch's forward Fisher-Yates shuffle by deterministic reservations (lb2_randperm).  Only numpy's legacy
RandomState (and the np.random global) is reproduced; np.random.Generator draws from PCG64 and is refused.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib

MT_N = 624

# torch's CPU generator state (torch.get_rng_state(), CPUGeneratorImplState): the seed at byte 0, `left` (int32) at 8, `next` (uint64)
# at 16, the 624 MT19937 words as uint64 from 24, the cached normals after them.  The next word is state[next] unless --left == 0,
# which twists first; between twists left + next == 625 (a fresh manual_seed has left 1, next 0).
TORCH_STATE_BYTES = 5056
_LEFT, _NEXT, _KEY = 8, 16, 24


def torch_state_decode(state: torch.Tensor) -> tuple[np.ndarray, int]:
    """(the 624 uint32 MT19937 words, numpy-convention position in [1, 624]) of a torch CPU generator state"""
    b = state.numpy() if isinstance(state, torch.Tensor) else np.asarray(state)
    if b.dtype != np.uint8 or b.shape != (TORCH_STATE_BYTES,):
        raise ValueError(f"torch generator state: expected {TORCH_STATE_BYTES} bytes (MT19937 CPU generator), got {b.dtype} {b.shape}")
    left = int(np.frombuffer(b[_LEFT:_LEFT + 4].tobytes(), "<i4")[0])
    nxt = int(np.frombuffer(b[_NEXT:_NEXT + 8].tobytes(), "<u8")[0])
    key64 = np.frombuffer(b[_KEY:_KEY + 8 * MT_N].tobytes(), "<u8")
    if not 1 <= left <= MT_N or (left > 1 and nxt != MT_N + 1 - left) or (key64 >> 32).any():
        raise ValueError(f"torch generator state: unknown layout (left {left}, next {nxt})")
    return key64.astype(np.uint32), MT_N + 1 - left


def torch_state_encode(state: torch.Tensor, key: np.ndarray, pos: int) -> torch.Tensor:
    """`state` with its MT19937 words and position replaced (every other field kept)"""
    b = state.numpy().copy()
    if b.shape != (TORCH_STATE_BYTES,):
        raise ValueError(f"torch generator state: expected {TORCH_STATE_BYTES} bytes, got {b.shape}")
    if not 1 <= pos <= MT_N:
        raise ValueError(f"position {pos} outside [1, {MT_N}]")
    b[_LEFT:_LEFT + 4] = np.frombuffer(np.array([MT_N + 1 - pos], "<i4").tobytes(), np.uint8)
    b[_NEXT:_NEXT + 8] = np.frombuffer(np.array([pos], "<u8").tobytes(), np.uint8)
    b[_KEY:_KEY + 8 * MT_N] = np.frombuffer(np.asarray(key, np.uint32).astype("<u8").tobytes(), np.uint8)
    return torch.from_numpy(b)


def untemper(w: np.ndarray) -> np.ndarray:
    """the MT19937 state words behind tempered outputs (tempering is a bijection of 32-bit words)"""
    y = np.asarray(w, np.uint32).astype(np.uint64)
    m32 = np.uint64(0xFFFFFFFF)
    y ^= y >> np.uint64(18)
    y ^= (y << np.uint64(15)) & np.uint64(0xEFC60000)
    x = y.copy()
    for _ in range(4):
        x = y ^ ((x << np.uint64(7)) & np.uint64(0x9D2C5680))
    y = x & m32
    y ^= (y >> np.uint64(11)) ^ (y >> np.uint64(22))
    return (y & m32).astype(np.uint32)


def _random_state(random_state):
    if random_state is None:
        return np.random.mtrand._rand
    if isinstance(random_state, np.random.Generator):
        raise TypeError("numpy_randn reproduces the legacy np.random.RandomState stream only; numpy.random.Generator (PCG64 / "
                        "ziggurat) is not supported")
    if not isinstance(random_state, np.random.RandomState):
        raise TypeError(f"random_state must be a numpy.random.RandomState, not {type(random_state).__name__}")
    return random_state


def _words(h, key: np.ndarray, pos: int, n: int):
    """(device uint32 words as int32, device state after them, position after them)"""
    state = torch.from_numpy(np.ascontiguousarray(key, np.uint32).view(np.int32)).to(h.device)
    words = torch.empty(max(n, 4), dtype=torch.int32, device=h.device)
    return words, state, h.mt19937_words(state, pos, n, words)


def _state_after(key, pos, used, words, n_words, state):
    """numpy's (key, pos) after `used` of the n_words words drawn from (key, pos): the block holding the last used word, untempered
    from `words` when it was emitted whole, else the generator's final block `state`"""
    first = MT_N - pos
    if used <= first:
        return key, pos + used
    twists = -(-(used - first) // MT_N)
    b = first + (twists - 1) * MT_N
    if b + MT_N <= n_words:
        return untemper(words[b:b + MT_N].cpu().numpy().view(np.uint32)), used - b
    return state.cpu().numpy().view(np.uint32).copy(), used - b


def _attempts(pairs: int) -> int:
    """attempts drawn for `pairs` accepted ones: acceptance is pi/4 per attempt, so the mean and 8 standard deviations (the rare
    shortfall draws more words of the stream)"""
    return math.ceil(pairs * 4 / math.pi + 8 * math.sqrt(pairs) + 16) if pairs else 0


def numpy_randn(*shape, device="cuda", random_state=None, band: float = _lib.GAUSS_BAND, stats: dict | None = None) -> torch.Tensor:
    """np.random.randn(*shape) (or random_state.randn) as an fp64 tensor on `device`, bit for bit; the generator's state afterwards
    (key, pos, has_gauss, cached gaussian) is what the host call leaves.  `band` (ulp) selects which logs the host resolves (0.5:
    all); `stats` (optional) receives the words, attempts and host-resolved logs."""
    rs = _random_state(random_state)
    name, key, pos, has_gauss, gauss = rs.get_state(legacy=True)
    if name != "MT19937":
        raise ValueError(f"numpy_randn: unknown bit generator {name}")
    shape = tuple(int(s) for s in shape)
    if any(s < 0 for s in shape):
        raise ValueError(f"negative dimensions are not allowed: {shape}")
    n = math.prod(shape)
    h = _lib.get_handle(device)
    out = torch.empty(max(n, 1), dtype=torch.float64, device=h.device)
    pairs = max(n - int(has_gauss), 0) + 1 >> 1
    n_words = 4 * _attempts(pairs)
    words, state, pos_end = _words(h, key, pos, n_words)
    while True:
        info = h.legacy_gauss(words, n_words, n, has_gauss, gauss, band, out)
        if not info.short_words:
            break
        more = max(n_words // 8, 4096)
        w2, state2, pos_end = _words(h, state.cpu().numpy().view(np.uint32), pos_end, more)
        words, state, n_words = torch.cat([words[:n_words], w2[:more]]), state2, n_words + more
    key2, pos2 = _state_after(key, pos, info.words_used, words, n_words, state)
    rs.set_state(("MT19937", np.asarray(key2, np.uint32), int(pos2), int(info.has_gauss), float(info.gauss)))
    if stats is not None:
        stats.update(words=int(info.words_used), attempts=int(info.words_used) // 4, pairs=pairs, deferred=int(info.deferred))
    return out[:n].view(shape)


def torch_randperm(n: int, device="cuda", generator: torch.Generator | None = None, stats: dict | None = None) -> torch.Tensor:
    """torch.randperm(n) of the CPU default generator (or the CPU `generator`) as an int64 tensor on `device`, bit for bit; the
    generator's state afterwards is what the host call leaves.  `stats` (optional) receives the reservation rounds."""
    g = torch.default_generator if generator is None else generator
    if g.device.type != "cpu":
        raise ValueError("torch_randperm reproduces torch's CPU generator; pass a CPU torch.Generator")
    n = int(n)
    if n < 0:
        raise ValueError(f"randperm: n must be >= 0, got {n}")
    if n >= _lib.RANDPERM_MAX_N:
        raise ValueError(f"randperm: n = {n} >= 2^32 / 20, where torch draws 64-bit words; not reproduced")
    h = _lib.get_handle(device)
    out = torch.empty(n, dtype=torch.int64, device=h.device)
    rounds = torch.zeros(1, dtype=torch.int32, device=h.device)
    if n < 2:                                      # torch draws no word
        h.randperm(None, n, out, rounds)
    else:
        s = g.get_state()
        key, pos = torch_state_decode(s)
        words, state, pos2 = _words(h, key, pos, n - 1)
        h.randperm(words, n, out, rounds)
        g.set_state(torch_state_encode(s, state.cpu().numpy().view(np.uint32), pos2))
    if stats is not None:
        stats.update(rounds=int(rounds.item()))
    return out
