"""CPU tests of the prompt step and the fork: the C entry qs_kv_cache_fork is exported with its documented signature, and the host checks of
backend.kv_cache_fork and of the prompt step's plan (qserve_b200.decode.prompt_pieces, which DecodeRunner.prefill runs before any launch)
reject bad arguments."""
import ctypes

import pytest
import torch


def test_kv_cache_fork_is_exported():
    from qserve_b200 import _lib

    P, I = ctypes.c_void_p, ctypes.c_int
    assert _lib.SIGNATURES["qs_kv_cache_fork"] == (ctypes.c_int, [P, P, P, P, I, I, I, I, I, I, I, I, P])
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "qs_kv_cache_fork")


def test_kv_cache_fork_rejects_bad_pairs_on_the_host():
    from qserve_b200 import backend

    table = torch.zeros((2, 4, 2, 3), dtype=torch.int64)  # [L, B, 2, blocks], never dereferenced: every call fails before a launch
    lens = torch.zeros(4, dtype=torch.int32)
    call = lambda parents, children: backend.kv_cache_fork(table, parents, children, lens, 2, 64, 128, True)
    with pytest.raises(RuntimeError, match="also a child"):
        call([0, 1], [1, 2])
    with pytest.raises(RuntimeError, match="appears twice"):
        call([0, 0], [2, 2])
    with pytest.raises(RuntimeError, match=r"\[0, 4\)"):
        call([0], [4])
    with pytest.raises(RuntimeError, match="children"):
        call([0, 1], [2])
    with pytest.raises(RuntimeError, match="CUDA"):  # valid pairs: the tensor checks come next
        call([0, 0], [1, 2])


def test_prompt_pieces_plan():
    from qserve_b200.decode import prompt_pieces

    lens = [1, 63, 64, 65, 130]
    assert prompt_pieces(lens, 130, 323) == [(0, lens)]
    assert prompt_pieces(lens, 130, 256, chunk=64) == [(0, [1, 63, 64, 64, 64]), (64, [0, 0, 0, 1, 64]), (128, [0, 0, 0, 0, 2])]
    assert [c for _, c in prompt_pieces([3, 1], 8, 2, chunk=1)] == [[1, 1], [1, 0], [1, 0]]


def test_prompt_pieces_rejects_bad_arguments():
    from qserve_b200.decode import prompt_pieces

    with pytest.raises(RuntimeError, match="ctx"):
        prompt_pieces([10, 101], 100, 4096)
    with pytest.raises(RuntimeError, match="ctx"):
        prompt_pieces([10, 0], 100, 4096)
    with pytest.raises(RuntimeError, match="chunk"):
        prompt_pieces([10, 20], 100, 4096, chunk=0)
    with pytest.raises(RuntimeError, match="prompt_tokens"):
        prompt_pieces([100, 100], 100, 199)
    with pytest.raises(RuntimeError, match="prompt_tokens"):
        prompt_pieces([100, 100], 100, 127, chunk=64)
    assert len(prompt_pieces([100, 100], 100, 128, chunk=64)) == 2
