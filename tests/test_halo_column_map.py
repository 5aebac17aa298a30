"""CPU checks of the K-halo column ownership (csrc/kernels/halo_columns.h): the same integer functions the stencil
kernel's loops call, evaluated on the host through the extension.  The map takes the launch geometry only (no rank,
no step), so it is the same on every rank and in every step; checked here: every float4 of a launch's column range
is visited by exactly one (CTA, thread), nothing outside the range is, and the owner function agrees with the loops."""
from hypothesis import given, settings, strategies as st

import hpc_patterns_b200


def host_chunks(tiles, chunks=16, max_sets=16):
    """[tile_begin, tile_end) ranges as HaloStencil.step_from_host cuts a row (one launch per range)."""
    chunks = max(1, min(chunks, tiles, max_sets))
    per = (tiles + chunks - 1) // chunks
    return [(k * per, min(tiles, (k + 1) * per)) for k in range(chunks) if k * per < tiles]


def check_launch(C, row_vec, tile_vec, t0, t1, ctas, threads):
    owner = {}
    for cta in range(ctas):
        for t in range(threads):
            for v in C.halo_thread_columns(row_vec, tile_vec, t0, t1, ctas, threads, cta, t):
                assert v not in owner, f"float4 {v} visited by {owner[v]} and {(cta, t)}"
                owner[v] = (cta, t)
    lo, hi = t0 * tile_vec, min(row_vec, t1 * tile_vec)
    assert set(owner) == set(range(lo, hi))
    for v in range(row_vec):
        assert C.halo_column_owner(row_vec, tile_vec, t0, t1, ctas, threads, v) == owner.get(v, (-1, -1))


@given(row_vec=st.integers(1, 3000), tile_kb=st.integers(1, 4), ctas=st.integers(1, 40), chunked=st.booleans())
@settings(max_examples=40, deadline=None)
def test_every_float4_has_exactly_one_owner(row_vec, tile_kb, ctas, chunked):
    """Whole-row launches and step_from_host's column chunks, 1 CTA up to more CTAs than tiles, the kernel's threads."""
    C = hpc_patterns_b200.native()
    tile_vec = tile_kb * 1024 // 16
    tiles = (row_vec + tile_vec - 1) // tile_vec
    for t0, t1 in host_chunks(tiles) if chunked else [(0, tiles)]:
        check_launch(C, row_vec, tile_vec, t0, t1, ctas, C.HALO_THREADS)


@given(row_vec=st.integers(1, 400), tile_vec=st.integers(1, 40), ctas=st.integers(1, 12), threads=st.integers(1, 16),
       data=st.data())
@settings(max_examples=60, deadline=None)
def test_any_sub_range_any_block_size(row_vec, tile_vec, ctas, threads, data):
    """Small tiles and blocks: tiles shorter than the block, ragged last tiles, arbitrary [tile_begin, tile_end)."""
    C = hpc_patterns_b200.native()
    tiles = (row_vec + tile_vec - 1) // tile_vec
    t0 = data.draw(st.integers(0, tiles - 1))
    t1 = data.draw(st.integers(t0 + 1, tiles))
    check_launch(C, row_vec, tile_vec, t0, t1, ctas, threads)


def test_last_tile_of_one_float4():
    C = hpc_patterns_b200.native()
    tile_vec = 1024 // 16
    check_launch(C, 5 * tile_vec + 1, tile_vec, 0, 6, 4, C.HALO_THREADS)
    assert C.halo_column_owner(5 * tile_vec + 1, tile_vec, 0, 6, 4, C.HALO_THREADS, 5 * tile_vec) == (1, 0)
