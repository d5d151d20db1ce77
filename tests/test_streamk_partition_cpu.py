"""Host-side model of the stream-K work partition of the persistent GEMM (pfd_b200/csrc/gemm_tc.cu: sk_range /
gemm_work<true> / the owner's contributor scan in sk_gather): the arithmetic is restated here 1:1 and checked
exhaustively over the tile counts, grid sizes and K depths the library can select, for the properties the device code
relies on.  (The device code itself is exercised by tests/test_kernels_gpu.py::test_gemm_stream_k_tail.)

Properties:
  * every (tail tile, K block) unit is processed exactly once; whole tiles exactly once;
  * a CTA has at most two segments, the head part of the next tile (contributor) comes first;
  * exactly one segment per tail tile reaches the last K block (the owner), it is mode 0 iff it also starts at block 0;
  * the owner's backwards scan finds exactly the contributors of its tile, each with the slot that contributor wrote
    (2c for a range that starts inside the tile, 2c + 1 for the spill-over from the previous tile), at most 6 of them
    under the host's admission rule R * 6 >= G;
  * dependencies only point to lower CTA indices and contributors wait for nobody (no cycles).
"""
import pytest


def sk_range(R, KB, c, G):
    U = R * KB
    return U * c // G, U * (c + 1) // G


def gemm_work(c, wi, G, dp_tiles, R, KB):
    """-> None or dict(tile, kb0, kb1, mode, slot); mirrors gemm_work<true> with sk_R > 0."""
    u0, u1 = sk_range(R, KB, c, G)
    t0 = u0 // KB
    aend = min(u1, (t0 + 1) * KB)
    has_b = u1 > aend
    nseg = (2 if has_b else 1) if u1 > u0 else 0
    if wi >= nseg:
        n_dp = dp_tiles // G
        if wi - nseg >= n_dp:
            return None
        return dict(tile=c + (wi - nseg) * G, kb0=0, kb1=KB, mode=0, slot=0)
    if wi == 0 and has_b:
        s0, s1, t = aend, u1, t0 + 1
    else:
        s0, s1, t = u0, aend, t0
    kb0, kb1 = s0 - t * KB, s1 - t * KB
    mode = (0 if kb0 == 0 else 2) if kb1 == KB else 1
    return dict(tile=dp_tiles + t, kb0=kb0, kb1=kb1, mode=mode, slot=2 * c + (1 if (wi == 0 and has_b) else 0))


def owner_sources(c, t, G, R, KB):
    """Contributor slots found by the owner's backwards scan (sk_gather, mode 2)."""
    tstart = t * KB
    out = []
    cc = c - 1
    while cc >= 0 and len(out) < 6:
        u0, u1 = sk_range(R, KB, cc, G)
        if u1 <= tstart:
            break
        if u1 > u0:
            out.append(2 * cc if u0 >= tstart else 2 * cc + 1)
        cc -= 1
    return out


@pytest.mark.parametrize("G", [148, 132, 8])
@pytest.mark.parametrize("KB", [16, 20, 45, 135, 270])
def test_stream_k_partition_properties(G, KB):
    for T in list(range(1, 3 * G + 2, max(1, G // 37))) + [128, 256, 512, 2 * G + 1]:
        R = T % G
        if R == 0 or R * 6 < G:                       # host admission rule (launch_gemm)
            continue
        dp_tiles = T - R
        units = {}                                    # (tile, kb) -> count
        written = {}                                  # slot -> (cta, tile)
        owners = {}
        for c in range(G):
            items = []
            wi = 0
            while True:
                w = gemm_work(c, wi, G, dp_tiles, R, KB)
                if w is None:
                    break
                items.append(w)
                wi += 1
            segs = [w for w in items if w["tile"] >= dp_tiles]
            assert len(segs) <= 2 and items[:len(segs)] == segs, "stream-K segments come first"
            if len(segs) == 2:
                assert segs[0]["mode"] == 1 and segs[0]["kb0"] == 0, "the head part of the next tile is a pure contributor"
                assert segs[1]["tile"] + 1 == segs[0]["tile"] and segs[1]["kb1"] == KB
            for w in items:
                assert 0 <= w["kb0"] < w["kb1"] <= KB and w["tile"] < T
                for kb in range(w["kb0"], w["kb1"]):
                    units[(w["tile"], kb)] = units.get((w["tile"], kb), 0) + 1
                if w["mode"] == 1:
                    assert w["slot"] not in written, "one writer per partial-tile slot"
                    written[w["slot"]] = (c, w["tile"])
                if w["tile"] >= dp_tiles and w["kb1"] == KB:
                    assert w["tile"] not in owners, "one owner per tail tile"
                    owners[w["tile"]] = (c, w)
                    assert (w["mode"] == 0) == (w["kb0"] == 0)
        assert len(units) == T * KB and set(units.values()) == {1}, "every K block of every tile exactly once"
        assert set(owners) == set(range(dp_tiles, T))
        for tile, (c, w) in owners.items():
            srcs = owner_sources(c, tile - dp_tiles, G, R, KB) if w["mode"] == 2 else []
            expect = sorted(s for s, (cc, tl) in written.items() if tl == tile)
            assert sorted(srcs) == expect, (T, G, KB, tile, srcs, expect)
            assert len(srcs) <= 6
            assert all(s // 2 < c for s in srcs), "dependencies point to lower CTA indices only"
        assert all(tl >= dp_tiles for _, tl in written.values())
