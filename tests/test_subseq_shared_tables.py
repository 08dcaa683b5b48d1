"""What the GPU tests of the sub-sequence decoder's one-thread finish (tests/test_gpu_subseq_finish.py) rest on, without a GPU:
the host model of k_huff_decode_subseq (tests/test_subseq_model.py) at the kernel's own constants, read from its sources,
reports the finish and the segments it takes on every stream whose components share one Huffman table set
(tests/_shared_tables.py), and gives the oracle's coefficients -- those of the standard-table stream of the same image."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _oracle as o  # noqa: E402
import _shared_tables as S  # noqa: E402
import test_subseq_model as M  # noqa: E402


@pytest.mark.parametrize("name", sorted(S.SHARED))
def test_model_reaches_the_finish(name):
    spec, (rounds, finished) = S.SHARED[name]
    jpeg, std = S.stream(*spec)
    want = o.coefficients(std)
    assert np.array_equal(o.coefficients(jpeg), want)
    if spec[6] == "one_id":
        assert not np.array_equal(jpeg, S.stream(*spec[:6], "shared")[0])
    got, cext, rep = M.model_decode(jpeg, sub_bytes=S.SUB_BYTES, warm_bits=S.WARM_BITS, rounds=S.ROUNDS)
    assert np.array_equal(got, want) and np.all(cext == 8), name
    segments = o.probe(jpeg).segment_count
    print("%s: %d bytes, %d segments, rounds %d, sub-sequences %d, finished by one thread %d" % (
        name, jpeg.size, segments, rep[0], rep[1], rep[2]))
    assert (rep[0] <= S.ROUNDS) if rounds is None else (rep[0] == rounds), name
    assert rep[2] == finished, name
    if spec[5]:   # a restart interval: some segments converge, some are finished
        assert 0 < finished < segments
    if rep[2]:    # the finish's output crosses tiles of 256 sub-sequences in the prefix phase
        assert rep[1] > 256
    assert jpeg.size < 100_000


def test_model_sub_sequence_sizes():
    """the sizes tests/test_gpu_subseq_finish.py sets with GPUJPEG_B200_SUBSEQ_BYTES: the minimum finishes, 1 KB converges"""
    jpeg, std = S.stream(*S.SHARED[S.SUB_SIZE_FRAME][0])
    want = o.coefficients(std)
    for sub, rounds in S.SUB_SIZES:
        got, _, rep = M.model_decode(jpeg, sub_bytes=sub, warm_bits=S.WARM_BITS, rounds=S.ROUNDS)
        assert np.array_equal(got, want)
        assert rep[0] == rounds and rep[2] == (rounds > S.ROUNDS), (sub, rep[:3])
