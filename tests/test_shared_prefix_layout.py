"""CPU tests of the shared-prefix layout: backend.shared_prefix_layout (tensors, offsets, host checks), the C entry's exported signature, and
the runner's group bookkeeping across fork -> fork -> prefill (decode.fork_groups) and its routing rule (decode.shared_prefix_route)."""
import ctypes

import pytest
import torch

from qserve_b200 import _lib
from qserve_b200 import backend as ext
from qserve_b200.decode import SHARED_PREFIX_MIN_PAGES, SHARED_PREFIX_MIN_ROWS, fork_groups, shared_prefix_route


def test_exported_signature():
    P, I, L, F, Z = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_size_t
    assert _lib.ABI_VERSION == 3
    assert _lib.SIGNATURES["qs_shared_prefix_decode_attention"] == (
        ctypes.c_int, [P, P, P, L, L, L] + [P] * 10 + [I] * 9 + [F, I, I, I, I, P, Z, P])
    assert _lib.SIGNATURES["qs_shared_prefix_attention_workspace_bytes"] == (ctypes.c_size_t, [I] * 8)


def test_layout_hand_case():
    lay = ext.shared_prefix_layout([[5, 1], [0], [2, 7, 3]], [3, 0, 16], batch=9)
    assert lay.group_offsets.tolist() == [0, 2, 3, 6]
    assert lay.group_rows.tolist() == [5, 1, 0, 2, 7, 3]
    assert lay.group_pages.tolist() == [3, 0, 16]
    assert lay.row_pages.tolist() == [0, 3, 16, 16, 0, 3, 0, 16, 0]
    assert (lay.num_groups, lay.max_group, lay.max_pages) == (3, 3, 16)
    assert all(t.dtype == torch.int32 and t.is_contiguous() for t in lay[:4])


def test_layout_empty():
    lay = ext.shared_prefix_layout([], [], batch=4)
    assert lay.group_offsets.tolist() == [0] and lay.group_rows.numel() == 0 and lay.row_pages.tolist() == [0] * 4
    assert (lay.num_groups, lay.max_group, lay.max_pages) == (0, 0, 0)


@pytest.mark.parametrize("groups,pages", [
    ([[0, 4]], [1]),          # row out of range
    ([[-1, 1]], [1]),         # negative row
    ([[0, 1], [1, 2]], [1, 1]),  # a row in two groups
    ([[0, 0]], [1]),          # a row twice in one group
    ([[0], []], [1, 1]),      # an empty group
    ([[0, 1]], [-1]),         # negative S
    ([[0, 1]], [1, 2]),       # one S per group
])
def test_layout_rejects(groups, pages):
    with pytest.raises(RuntimeError):
        ext.shared_prefix_layout(groups, pages, batch=4)


def test_fork_fork_prefill_bookkeeping():
    cached = [200, 0, 0, 0, 130, 0, 64, 0]
    g = fork_groups([], [0, 0, 0], [1, 2, 3], cached)
    assert g == [((0, 1, 2, 3), 3)]
    # a second fork with another parent: a new group, the first one stays
    g = fork_groups(g, [4], [5], cached)
    assert g == [((0, 1, 2, 3), 3), ((4, 5), 2)]
    # a fork that touches a member dissolves that member's group
    cached[2] = 300
    g = fork_groups(g, [2], [7], cached)
    assert g == [((4, 5), 2), ((2, 7), 4)]
    # two parents in one fork: one group each
    g2 = fork_groups(g, [6, 4, 6], [1, 0, 3], cached)
    assert g2 == [((2, 7), 4), ((6, 1, 3), 1), ((4, 0), 2)]
    # prefill dissolves everything (the runner sets []), and the layout of any bookkeeping result passes the host checks
    for gr in (g, g2):
        ext.shared_prefix_layout([r for r, _ in gr], [s for _, s in gr], batch=8)


def test_route_rule():
    assert not shared_prefix_route([])
    assert not shared_prefix_route([((0,), 50)])
    small = max(SHARED_PREFIX_MIN_ROWS - 1, 1)
    assert not shared_prefix_route([(tuple(range(small)), SHARED_PREFIX_MIN_PAGES)]) or small >= SHARED_PREFIX_MIN_ROWS
    assert not shared_prefix_route([(tuple(range(SHARED_PREFIX_MIN_ROWS)), SHARED_PREFIX_MIN_PAGES - 1)])
    assert shared_prefix_route([((9,), 0), (tuple(range(SHARED_PREFIX_MIN_ROWS)), SHARED_PREFIX_MIN_PAGES)])
