"""CPU checks of the shared-memory images the decoder-layer kernels (mlp_tc.cu) hand to wgmma, with the address helpers and the
descriptor builder lifted from the product sources.

The tensor cores read a K-major SWIZZLE_128B operand from a descriptor: start address >> 4, stride byte offset (SBO) between 8-row
atoms, swizzle mode; inside an 8-row atom, row n lies n * 128 bytes from the start and the hardware XORs address bits 4-6 with bits
7-9.  `read_addr` below emulates that address generation; every element a wgmma k-step reads must be the element the producer wrote
there (and that the epilogue reads back)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gaussianavatar_b200", "csrc")


def _py(expr: str) -> str:
    """A C expression turned into Python (casts and integer suffixes dropped)."""
    expr = re.sub(r"\((?:uint32_t|uint64_t)\)", "", expr)
    return re.sub(r"\b(0[xX][0-9A-Fa-f]+|\d+)u\b", r"\1", expr)


def _lift(src: str, ret: str, name: str, args: str):
    m = re.search(r"__device__ __forceinline__ " + ret + r" " + name + r"\(([^)]*)\)\s*\{\s*return (.*?);\s*\}", src, re.S)
    assert m, name
    params = [a.split()[-1] for a in m.group(1).split(",")]
    assert params == args.split(), (name, params)
    return _py(m.group(2))


TCC = open(os.path.join(CSRC, "tc_common.cuh")).read()
MLP = open(os.path.join(CSRC, "mlp_tc.cu")).read()
_SW = _lift(TCC, "uint32_t", "sw128_offset", "r u")
_KM = _lift(TCC, "uint32_t", "kmajor_off", "r k chunk_bytes")
_DESC = _lift(TCC, "uint64_t", "wgmma_desc", "saddr")
_KSTEP = _lift(TCC, "uint32_t", "kstep_addr", "base ks chunk_bytes")


def sw128_offset(r, u):
    return eval(_SW, {}, dict(r=r, u=u))


def kmajor_off(r, k, chunk_bytes):
    return eval(_KM, {"sw128_offset": sw128_offset}, dict(r=r, k=k, chunk_bytes=chunk_bytes))


def wgmma_desc(saddr):
    return eval(_DESC, {}, dict(saddr=saddr))


def kstep_addr(base, ks, chunk_bytes):
    return eval(_KSTEP, {}, dict(base=base, ks=ks, chunk_bytes=chunk_bytes))


def read_addr(desc, n, kk):
    """Shared-memory byte address of element (row n, k = kk of the k-step) that wgmma reads for a TF32 K-major SWIZZLE_128B descriptor."""
    assert desc >> 62 == 1, "swizzle mode 128 B"
    start = (desc & 0x3FFF) << 4
    sbo = ((desc >> 32) & 0x3FFF) << 4
    lin = start + (n // 8) * sbo + (n % 8) * 128 + kk * 4
    return lin ^ (((lin >> 7) & 7) << 4)


def test_wgmma_descriptor_fields():
    for saddr in (0, 1024, 0x8400 + 32, 0x8400 + 96, 227 * 1024 - 1024):
        d = wgmma_desc(saddr)
        assert d < 1 << 64
        assert d & 0x3FFF == saddr >> 4                       # start address >> 4, bits 0-13
        assert (d >> 16) & 0x3FFF == 1                        # leading byte offset: unused by swizzled K-major layouts
        assert ((d >> 32) & 0x3FFF) << 4 == 1024              # SBO: 8 rows of 128 B
        assert (d >> 49) & 7 == 0                             # base offset: images start on 1024-byte boundaries
        assert d >> 62 == 1                                   # SWIZZLE_128B
        assert d & ~((0x3FFF) | (0x3FFF << 16) | (0x3FFF << 32) | (7 << 49) | (3 << 62)) == 0
    for ks in range(16):                                      # k-step advance: 32 bytes inside the 128-byte row, then the next chunk
        assert kstep_addr(0, ks, 8192) == (ks // 4) * 8192 + (ks % 4) * 32
    assert [kstep_addr(4096, ks, 0) for ks in range(4)] == [4096, 4128, 4160, 4192]


def _check_image(base, rows, ksteps, chunk_bytes):
    """Every element of every k-step of a K-major image is read where kmajor_off (the producers' layout) puts it."""
    seen = set()
    for ks in range(ksteps):
        d = wgmma_desc(kstep_addr(base, ks, chunk_bytes))
        for n in range(rows):
            for kk in range(8):
                got = read_addr(d, n, kk) - base
                assert got == kmajor_off(n, 8 * ks + kk, chunk_bytes), (rows, ks, n, kk)
                seen.add(got)
    assert seen == set(range(0, rows * 4 * ksteps * 8, 4))


def test_wgmma_reads_the_forward_and_backward_images():
    _check_image(0x8000 + 3 * 32768, 64, 16, 64 * 128)        # forward: X tile, N = 64 pixels, K = 128 in 8 KB chunks
    _check_image(0x8000 + 2 * 16384, 32, 16, 32 * 128)        # backward data gradient: G tile, N = 32 pixels, K = 128 output channels
    _check_image(0x10000 + 16384, 128, 4, 0)                  # backward weight gradient: transposed X, N = 128 channels, K = 32 pixels


def test_tc_bwd_transposed_x_writes():
    """Backward producer (warp w = 0..3, lane): after the producer barrier, thread (w, lane) converts the 4-pixel x 4-channel blocks
    pixels 4 q .. 4 q + 3 (q = lane / 4), channels 4 cg .. 4 cg + 3 (cg = 4 (2 w + b) + lane % 4, b = 0, 1), reading them from the
    pixel-major image (`mnmajor_off`) and writing channel c's four pixels as the 16-byte piece `sw128_offset(c, q)` of the transposed
    image, as lifted from mlp_tc.cu.  The blocks must cover the 32-pixel x 128-channel tile exactly once, each pixel must land where the
    weight-gradient wgmma and the epilogue read it (`kmajor_off(c, px, 0)`), and each warp instruction of the transposed writes must
    spread its 16-byte pieces evenly over the 32 banks."""
    assert "cgs[b] = 4 * (2 * warp + b) + (lane & 3)" in MLP and "const int q = lane >> 2;" in MLP
    assert "mnmajor_off(4 * q + r, c0, kGkChunk)" in MLP and "const int c0 = 4 * cgs[b];" in MLP
    for i in range(4):
        assert f"sw128_offset(c0 + {i}, q)" in MLP
    blocks, seen_xt = set(), set()
    for warp in range(4):
        inst_xt = {}
        for lane in range(32):
            q = lane >> 2
            for b in range(2):
                cg = 4 * (2 * warp + b) + (lane & 3)
                blocks.update((4 * q + r, 4 * cg + i) for r in range(4) for i in range(4))
                for i in range(4):                            # channel 4 cg + i, pixels 4 q .. 4 q + 3
                    c = 4 * cg + i
                    xo = sw128_offset(c, q)
                    for j in range(4):
                        assert xo + 4 * j == kmajor_off(c, 4 * q + j, 0), (warp, lane, b, i, j)
                    seen_xt.add(xo)
                    inst_xt.setdefault((b, i), []).append(xo)
        for offs in inst_xt.values():
            assert len(offs) == 32
            assert sorted((o % 128) // 16 for o in offs) == sorted(list(range(8)) * 4)   # 4 wavefronts: the minimum for 512 B
    assert blocks == {(px, c) for px in range(32) for c in range(128)}
    assert seen_xt == set(range(0, 16384, 16))
