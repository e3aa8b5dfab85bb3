"""CPU checks of the output staging of the decoder-layer kernels (mlp_tc.cu), with the address helper and the staging expressions
lifted from the product sources.

Each consumer warpgroup of `tc_fwd_kernel` / `tc_bwd_kernel` writes its accumulator fragments into its own staging half, two chunks
of 32 channels x `rows` pixels in the K-major layout (`kmajor_off`), and one thread moves each chunk with a TMA tensor store of a
SWIZZLE_128B box of 32 fp32 x `rows`.  In shared memory such a box lies row after row, 128 B per row, with the 16-byte unit index
XORed with the row index modulo 8 (address bits 4-6 XOR bits 7-9 of a 1024-byte-aligned box).  Every fragment element must sit where
the box expects it, a tile's writes must cover the staging exactly once, and each warp store must hit 32 distinct banks."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gaussianavatar_b200", "csrc")
TCC = open(os.path.join(CSRC, "tc_common.cuh")).read()
MLP = open(os.path.join(CSRC, "mlp_tc.cu")).read()


def _py(expr: str) -> str:
    expr = re.sub(r"\((?:uint32_t|uint64_t)\)", "", expr)
    return re.sub(r"\b(0[xX][0-9A-Fa-f]+|\d+)u\b", r"\1", expr)


def _lift(name: str, args: str) -> str:
    m = re.search(r"__device__ __forceinline__ uint32_t " + name + r"\(([^)]*)\)\s*\{\s*return (.*?);\s*\}", TCC, re.S)
    assert m, name
    assert [a.split()[-1] for a in m.group(1).split(",")] == args.split(), name
    return _py(m.group(2))


_SW, _KM = _lift("sw128_offset", "r u"), _lift("kmajor_off", "r k chunk_bytes")


def sw128_offset(r, u):
    return eval(_SW, {}, dict(r=r, u=u))


def kmajor_off(r, k, chunk_bytes):
    return eval(_KM, {"sw128_offset": sw128_offset}, dict(r=r, k=k, chunk_bytes=chunk_bytes))


def tma_box_addr(row, col):
    """Byte offset of element (row, col) of a 32-column fp32 SWIZZLE_128B box whose shared-memory base is 1024-byte aligned."""
    lin = row * 128 + col * 4
    return lin ^ (((lin >> 7) & 7) << 4)


def _check_staging(rows, ntiles, frag, chunk_name):
    """frag(warp, lane) yields (array slot, channel, pixel, staging-offset expression arguments) of every element the thread writes
    per tile; `rows` pixels per tile, staging halves of two chunks of rows x 128 B."""
    chunk = rows * 128
    seen = {0: [], 1: []}
    for warp in range(4, 12):
        wg = (warp - 4) >> 2
        per_inst = {}
        for lane in range(32):
            for slot, ch, px, chl in frag(warp, lane):
                assert 64 * wg <= ch < 64 * wg + 64 and chl == ch - 64 * wg
                off = kmajor_off(px, chl, chunk)
                c = chl // 32                                 # the chunk the TMA store of column 64 wg + 32 c moves
                assert off == c * chunk + tma_box_addr(px, chl % 32), (chunk_name, warp, lane, slot)
                seen[wg].append(off)
                per_inst.setdefault(slot, []).append(off)
        for slot, offs in per_inst.items():                    # one st.shared.b32 per slot: 32 lanes, 32 distinct banks
            assert len(offs) == 32
            assert len({(o // 4) % 32 for o in offs}) == 32, (chunk_name, warp, slot)
    for wg in (0, 1):
        assert sorted(seen[wg]) == list(range(0, 2 * chunk, 4)), chunk_name


def test_forward_staging_matches_the_tma_box():
    for s in ("const int oc = 16 * (warp - 4) + g;", "const int wg = (warp - 4) >> 2, ocl = oc - 64 * wg;",
              "kmajor_off(px, ocl, kTChunk)", "kmajor_off(px, ocl + 8, kTChunk)", "const int px = 8 * nt + 2 * t4 + e;",
              "tma_store_2d(&p.ymap, ys_u + c * kTChunk, 64 * wg + 32 * c, tile * kTPx)",
              "tma_load_2d(ys_u + c * kTChunk, &p.ymap, yload, 64 * wg + 32 * c, tile * kTPx)",
              "make_tmap(&p.ymap, Y, 128, M, ldy, kTPx)", "constexpr int kTPx = 64", "kTChunk = kTPx * 128"):
        assert s in MLP, s

    def frag(warp, lane):
        g, t4 = lane >> 2, lane & 3
        oc = 16 * (warp - 4) + g
        ocl = oc - 64 * ((warp - 4) >> 2)
        for nt in range(8):
            for e in range(2):
                px = 8 * nt + 2 * t4 + e
                yield (nt, e, 0), oc, px, ocl
                yield (nt, e, 1), oc + 8, px, ocl + 8
    _check_staging(64, 1, frag, "forward")


def test_backward_staging_matches_the_tma_box():
    for s in ("const int ic = 16 * (warp - 4) + g;", "const int wg = (warp - 4) >> 2, icl = ic - 64 * wg;",
              "kmajor_off(px, icl + 8 * h, kGkChunk)", "const int px = 8 * nt + 2 * t4 + e;", "const int c = ic + 8 * h;",
              "tma_store_2d(&p.omap, os_u + c * kGkChunk, 64 * wg + 32 * c, m0)",
              "tma_reduce_add_2d(&p.omap, os_u + c * kGkChunk, 64 * wg + 32 * c, m0)",
              "tma_load_2d(os_u + c * kGkChunk, &p.omap, oload, 64 * wg + 32 * c, m0)",
              "make_tmap(&p.omap, dZprev, kin, M, ldo, kPx)", "constexpr int kPx = 32;", "kGkChunk = kPx * 128"):
        assert s in MLP, s

    def frag(warp, lane):
        g, t4 = lane >> 2, lane & 3
        ic = 16 * (warp - 4) + g
        icl = ic - 64 * ((warp - 4) >> 2)
        for nt in range(4):
            for e in range(2):
                px = 8 * nt + 2 * t4 + e
                for h in range(2):
                    yield (nt, e, h), ic + 8 * h, px, icl + 8 * h
    _check_staging(32, 1, frag, "backward")


def test_backward_chunks_cover_the_valid_input_channels():
    """The chunks a warpgroup moves are those holding an input channel below kin (the tensor map clips the rest of a chunk)."""
    m = re.search(r"const int nchunks = (.*?);", MLP)
    assert m
    expr = m.group(1).replace("p.kin", "kin").replace("/", "//")
    for kin in range(4, 129, 4):
        moved = set()
        for wg in (0, 1):
            n = eval(expr, {"max": max, "min": min}, dict(kin=kin, wg=wg))
            assert 0 <= n <= 2
            moved |= {64 * wg + 32 * c for c in range(n)}
        assert moved == {c0 for c0 in range(0, 128, 32) if c0 < kin}, kin


def test_tensor_map_box_is_the_staging_chunk():
    assert "box[2] = {32, (cuuint32_t)box_rows}" in MLP
    assert "CU_TENSOR_MAP_SWIZZLE_128B" in MLP and "CU_TENSOR_MAP_DATA_TYPE_FLOAT32" in MLP
    assert re.search(r"unsigned char ys\[2\]\[2 \* kTChunk\];", MLP) and re.search(r"unsigned char os\[2\]\[2 \* kGkChunk\];", MLP)
