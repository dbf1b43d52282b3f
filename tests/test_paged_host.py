"""CPU tests of the paged KV cache's host side: PagePool's assignment, release, fork and reference counts, every failure leaving its
state unchanged, and the BatchDecoder(pages=...) rejections that need no device."""
import copy

import pytest

from squeezellm_b200.runtime import PAGE, PagePool


def state(pool):
    return copy.deepcopy((pool._free, pool.refs, pool.tables))


def test_assign_and_release():
    pool = PagePool(6, 3, 4)
    assert pool.free == 6 and pool.tables[0] == [-1] * 4
    assert pool.assign(0, 2) == [(0, 0), (1, 1)]
    assert pool.assign(0, 3) == [(2, 2)]          # only the missing block
    assert pool.assign(0, 3) == []
    assert pool.assign(1, 1) == [(0, 3)]
    assert pool.free == 2 and pool.held(0) == 3 and pool.refs[:4] == [1, 1, 1, 1]
    pool.release(0)
    assert pool.free == 5 and pool.tables[0] == [-1] * 4 and pool.held(0) == 0
    got = pool.assign(2, 4)                        # freed pages come back, in a different order
    assert [j for j, _ in got] == [0, 1, 2, 3] and sorted(p for _, p in got) == [0, 1, 2, 4] and pool.free == 1


def test_fresh_assign_drops_the_slot_pages_first():
    pool = PagePool(3, 2, 4)
    pool.assign(0, 3)
    assert pool.need(0, 3, fresh=True) == 0
    pool.assign(0, 3, fresh=True)
    assert pool.free == 0 and sorted(pool.tables[0][:3]) == [0, 1, 2]


def test_empty_pool_changes_nothing():
    pool = PagePool(3, 2, 4)
    pool.assign(0, 2)
    before = state(pool)
    with pytest.raises(RuntimeError, match=r"slot\(s\) \[1\]"):
        pool.assign(1, 2)
    assert state(pool) == before
    with pytest.raises(RuntimeError, match=r"slot\(s\) \[0, 1\]"):
        pool.reserve({0: (3, False), 1: (1, False)})
    assert state(pool) == before


def test_fork_shares_full_pages_and_copies_the_partial_one():
    pool = PagePool(8, 3, 4)
    pool.assign(0, 3)                              # position 130: blocks 0, 1 full, block 2 partial
    cp = pool.fork(0, 1, 130)
    assert pool.tables[1][:2] == pool.tables[0][:2] and pool.refs[0] == pool.refs[1] == 2
    assert cp == (pool.tables[0][2], pool.tables[1][2]) and pool.tables[1][2] not in pool.tables[0]
    pool.release(0)                                # the shared pages stay with slot 1
    assert pool.refs[0] == pool.refs[1] == 1 and pool.free == 8 - 3
    pool.release(1)
    assert pool.free == 8 and pool.refs == [0] * 8


def test_fork_at_a_page_boundary_copies_nothing():
    pool = PagePool(4, 2, 4)
    pool.assign(0, 2)
    assert pool.fork(0, 1, 2 * PAGE) is None
    assert pool.free == 2 and pool.tables[1][:2] == pool.tables[0][:2]


def test_fork_without_a_free_page_changes_nothing():
    pool = PagePool(2, 2, 4)
    pool.assign(0, 2)
    before = state(pool)
    with pytest.raises(RuntimeError, match="no free page"):
        pool.fork(0, 1, 70)
    assert state(pool) == before
    with pytest.raises(ValueError, match="already holds pages"):
        pool.fork(1, 0, 64)


def test_double_release_is_rejected():
    pool = PagePool(4, 2, 4)
    pool.assign(0, 2)
    pool.refs[pool.tables[0][0]] = 0               # as if the page had been let go already
    before = state(pool)
    with pytest.raises(ValueError, match="already free"):
        pool.release(0)
    assert state(pool) == before


pytest.importorskip("transformers")


@pytest.mark.parametrize("pages,frag", [(0, "1..2"), (3, "1..2"), (-1, "1..2"), (2.0, "got 2.0"), (True, "got True"), ("3", "got '3'")])
def test_decoder_rejects_bad_pages(pages, frag):
    from test_decoder_host import quantized
    from squeezellm_b200.runtime import BatchDecoder
    with pytest.raises(ValueError, match=f"pages must be None or an int in .*{frag}" if frag == "1..2" else f"pages .*{frag}"):
        BatchDecoder(quantized(), 64, 2, pages=pages)   # 2 slots x ceil(64 / 64) pages at most
