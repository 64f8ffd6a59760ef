"""Side notes of the keccak extension for the fill tests (tests/test_keccak_fill_cpu.py, tests/test_gpu_keccak_fill.py), and the finalize
permutation restated in numpy."""
import numpy as np

from nexus_zkvm_b200 import keccak as K


def edge_machine(n_perms, seed=0):
    """A KeccakMachine over an explicit side note with the edge cases of the fill: all-zero and all-ones input states, address low halves at
    0xFFFF - k (k < 200, so the carry crosses inside the 200 bytes), the largest address whose range does not wrap (2^32 - 200), timestamp low
    halves at 0xFFFF and the largest accepted timestamp (2^32 - 2)."""
    rng = np.random.default_rng(seed)
    inputs = rng.integers(0, 1 << 64, (n_perms, 25), dtype=np.uint64, endpoint=False)
    inputs[0::3] = 0
    inputs[1::3] = np.uint64((1 << 64) - 1)
    k = rng.integers(0, K.STATE_SIZE, n_perms)
    addresses = (rng.integers(0, 0xFFFF, n_perms).astype(np.uint64) << np.uint64(16)) | (0xFFFF - k).astype(np.uint64)
    addresses[-1] = (1 << 32) - K.STATE_SIZE
    timestamps = rng.integers(0, (1 << 32) - 1, (n_perms, K.STATE_SIZE), dtype=np.uint64)
    timestamps[:, 1::2] = (((timestamps[:, 1::2] >> np.uint64(16)) % np.uint64(0xFFFF)) << np.uint64(16)) | np.uint64(0xFFFF)
    timestamps[0, 0] = (1 << 32) - 2
    return K.KeccakMachine(inputs=inputs, addresses=addresses, timestamps=timestamps)


def finalized_src_rows(log_size):
    """Position i of a finalized column holds trace row src[i]: coset order -> circle-domain order -> bit reversal."""
    n = 1 << log_size
    i = np.arange(n, dtype=np.int64)
    j = np.zeros(n, np.int64)
    for b in range(log_size):
        j |= ((i >> b) & 1) << (log_size - 1 - b)
    half = n >> 1
    return np.where(j < half, 2 * j, n - 1 - 2 * (j - half))


def finalized_main_trace(m):
    """KeccakMachine.fill_main_trace() in finalized order, as the five batches nb200_keccak_main_trace returns (uint32)."""
    cols = m.fill_main_trace()
    blocks = [np.asarray(b, dtype=np.uint32) for b in cols[:3]]
    mults = [np.asarray(c, dtype=np.uint32) for c in cols[3:]]
    out = [b[:, finalized_src_rows(b.shape[1].bit_length() - 1)] for b in blocks]
    bitwise = np.stack(mults[:32])
    out.append(bitwise[:, finalized_src_rows(K.BITWISE_LOG_SIZE)])
    out.append(mults[32][None, finalized_src_rows(K.ROTATE_LOG_SIZE)])
    return out
