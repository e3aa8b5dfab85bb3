"""CPU checks of device-side math lifted from the product sources and compiled for the host (no GPU needed).

1. The sub-tile culling of the compositing kernels must be CONSERVATIVE -- a (Gaussian, sub-tile) pair may only be skipped when
every pixel of the sub-tile would have been skipped by the exact per-pixel test (alpha < 1/255 or power > 0) anyway; that is what makes
the culled kernels bit-identical to the un-culled algorithm.  The test lifts the source text of `cull_radius2` / `rect_dist2` out of
csrc/raster.cu, compiles it for the host and brute-forces random conics, opacities and rectangles (including extreme anisotropy)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <cmath>
#include <cstdio>
#include <cstdint>
struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
#define __device__
#define __forceinline__ inline
%(functions)s
static uint64_t s = 0x9E3779B97F4A7C15ull;
static inline double rnd() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (double)(s >> 11) / 9007199254740992.0; }
int main()
{
    long culled = 0, violations = 0, evaluated = 0;
    for (long it = 0; it < 400000; ++it) {
        // random 2D covariance: rotation angle, two axis lengths over six orders of magnitude of anisotropy (+0.3 dilation as in K1)
        const double th = rnd() * 3.14159265358979, l1 = std::exp(rnd() * 9.0 - 2.0), l2 = l1 * std::exp(-rnd() * 12.0);
        const double c = std::cos(th), sn = std::sin(th);
        const float a = (float)(c * c * l1 + sn * sn * l2 + 0.3), b = (float)(c * sn * (l1 - l2)), cc = (float)(sn * sn * l1 + c * c * l2 + 0.3);
        const float det = a * cc - b * b;
        if (!(det > 0.f)) continue;
        float4 co; co.x = cc / det; co.y = -b / det; co.z = a / det;
        co.w = (it %% 7 == 0) ? 1.0f : (float)std::exp(-rnd() * 8.0);            // opacity: 1 (the avatar's constant) or down to 3e-4
        const float rc2 = cull_radius2(co);
        const float reach = 4.f * std::sqrt((float)l1 + 0.3f) + 12.f;
        for (int k = 0; k < 8; ++k) {
            const int sx = (int)(rnd() * 1000), sy = (int)(rnd() * 1000);
            float2 ctr; ctr.x = (float)(sx + 3.5 + (rnd() * 2 - 1) * reach); ctr.y = (float)(sy + 1.5 + (rnd() * 2 - 1) * reach);
            const float d2 = rect_dist2(ctr, (float)sx, (float)(sx + 7), (float)sy, (float)(sy + 3));
            ++evaluated;
            if (!(d2 > rc2)) continue;                                            // the kernels evaluate this pair exactly
            ++culled;
            for (int py = sy; py < sy + 4; ++py)
                for (int px = sx; px < sx + 8; ++px) {
                    const float dx = ctr.x - (float)px, dy = ctr.y - (float)py;
                    const float power = -0.5f * (co.x * dx * dx + co.z * dy * dy) - co.y * dx * dy;
                    if (power > 0.f) continue;
                    const float alpha = std::fmin(0.99f, co.w * std::exp(power));
                    if (!(alpha < 1.0f / 255.0f)) ++violations;
                }
        }
    }
    std::printf("%%ld %%ld %%ld\n", evaluated, culled, violations);
    return 0;
}
"""


def _extract(src, name):
    m = re.search(r"__device__ __forceinline__ float " + name + r"\(.*?\n}\n", src, re.S)
    assert m, f"{name} not found in raster.cu"
    return m.group(0)


def test_subtile_culling_is_conservative(tmp_path):
    src = open(os.path.join(ROOT, "gaussianavatar_b200", "csrc", "raster.cu")).read()
    code = HARNESS % {"functions": _extract(src, "cull_radius2") + "\n" + _extract(src, "rect_dist2")}
    cpp, exe = tmp_path / "cull.cpp", tmp_path / "cull"
    cpp.write_text(code)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    for flags in (["-O2", "-ffp-contract=off"], ["-O2", "-ffp-contract=fast", "-march=native"]):
        r = subprocess.run([cxx, "-std=c++17", *flags, "-o", str(exe), str(cpp)], capture_output=True, text=True)
        if r.returncode != 0 and "-march=native" in flags:
            continue
        assert r.returncode == 0, r.stderr
        out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300).stdout.split()
        evaluated, culled, violations = (int(v) for v in out)
        assert evaluated > 1_000_000 and culled > 100_000, (evaluated, culled)   # the test really exercises the cull branch
        assert violations == 0, f"{violations} pixels of culled pairs would have been blended"


LAYOUT_HARNESS = r"""
#include <cstdio>
#include <cstdint>
#include <set>
#define __device__
#define __forceinline__ inline
%(functions)s
// byte offset of element (k, m) of the pixel-major image: 32-element chunks lbo apart, 4-row atoms sbo apart, 32-byte pieces XOR k %% 4
static uint32_t probe_byte(int k, int m, uint32_t lbo, uint32_t sbo)
{ return (uint32_t)(m / 32) * lbo + (uint32_t)(k / 4) * sbo + (uint32_t)(k %% 4) * 128u + (uint32_t)((((m %% 32) / 8) ^ (k %% 4)) * 32) + (uint32_t)(m %% 8) * 4u; }
int main()
{
    int bad = 0;
    std::set<uint32_t> seen;
    for (int r = 0; r < 32; ++r)                 // r = K index (pixel) inside a 32-row chunk, v = 16-byte unit = channels 4v..4v+3
        for (int v = 0; v < 8; ++v) {
            const uint32_t off = mn_unit(r, v);
            bad += off != probe_byte(r, 4 * v, 4096, 512);          // SBO = 512: 4-row atoms are contiguous, so row r sits at r * 128
            bad += (off %% 16) != 0 || off >= 4096;
            seen.insert(off);
        }
    bad += seen.size() != 256;                   // a bijection onto the chunk's 256 sixteen-byte slots
    seen.clear();
    for (int r = 0; r < 128; ++r)                // K-major 128-byte swizzle: 16-byte unit u of row r
        for (int u = 0; u < 8; ++u) {
            const uint32_t off = sw128_offset(r, u);
            bad += off != (uint32_t)r * 128u + (uint32_t)((u ^ (r & 7)) << 4);
            seen.insert(off);
        }
    bad += seen.size() != 1024;
    for (int r = 0; r < 32; ++r)                 // element offsets the MMA fragments are read with: the same images, word by word
        for (int c = 0; c < 128; ++c) {
            bad += mnmajor_off(r, c, 4096) != probe_byte(r, c, 4096, 512);
            bad += kmajor_off(r, c, 4096) != (uint32_t)(c / 32) * 4096u + sw128_offset(r, (c %% 32) / 4) + (uint32_t)(c %% 4) * 4u;
        }
    std::printf("%%d\n", bad);
    return 0;
}
"""


def test_umma_layout_helpers_match_the_decoded_hardware_layout(tmp_path):
    """`mn_unit`, `sw128_offset`, `kmajor_off` and `mnmajor_off` (tc_common.cuh), lifted from the product source and compiled for the
    host: the pixel-major helpers must reproduce that layout word by word, the K-major ones the 128-byte swizzle, and the piece helpers
    must be bijections onto their tiles."""
    tcc = open(os.path.join(ROOT, "gaussianavatar_b200", "csrc", "tc_common.cuh")).read()
    fs = [re.search(r"__device__ __forceinline__ uint32_t " + n + r"\(.*?\}\n", tcc, re.S) for n in ("sw128_offset", "kmajor_off", "mn_unit", "mnmajor_off")]
    assert all(fs)
    cpp, exe = tmp_path / "layout.cpp", tmp_path / "layout"
    cpp.write_text(LAYOUT_HARNESS % {"functions": "\n".join(f.group(0) for f in fs)})
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++17", "-O1", "-o", str(exe), str(cpp)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)], capture_output=True, text=True, timeout=60).stdout.strip() == "0"


def _c_expr(src: str, pattern: str) -> str:
    """One C initialiser lifted from the product source, turned into a Python expression (casts and integer suffixes dropped)."""
    m = re.search(pattern, src)
    assert m, pattern
    e = m.group(1)
    e = re.sub(r"\(uint32_t\)", "", e)
    e = re.sub(r"(\d+)u\b", r"\1", e)
    return e


def test_tc_bwd_piece_addresses_are_the_umma_images():
    """mlp_tc.cu, backward layer: the cp.async destinations / in-place conversion addresses of the converter threads (`k_off`, `mn_off`),
    lifted from the kernel source as written, and the element offsets the MMA fragments and the epilogue's read-back of x use
    (`kmajor_off`, `mnmajor_off`, lifted from tc_common.cuh), against the two image layouts: K-major with the 128-byte swizzle (16-byte
    units XOR px % 8) and pixel-major with 32-byte pieces XOR px % 4 (formula in the kernel's comment).  Every thread must own whole
    16-byte pieces, the pieces of one array must tile the 32-pixel x 128-channel image exactly once, and a read of element (px, c) must
    land where the conversion wrote it."""
    src = open(os.path.join(ROOT, "gaussianavatar_b200", "csrc", "mlp_tc.cu")).read()
    k_off = _c_expr(src, r"const uint32_t k_off = (.*?);\s")
    mn_off = _c_expr(src, r"const uint32_t mn_off = (.*?);\n")
    tcc = open(os.path.join(ROOT, "gaussianavatar_b200", "csrc", "tc_common.cuh")).read()
    kmaj = _c_expr(tcc, r"uint32_t kmajor_off\(int r, int k, uint32_t chunk_bytes\)\n\{\n\s*return (.*?);\n").replace("chunk_bytes", "kGkChunk")
    mnmaj = _c_expr(tcc, r"uint32_t mnmajor_off\(int k, int mn, uint32_t chunk_bytes\)\n\{\n\s*return (.*?);\n").replace("chunk_bytes", "kGkChunk")
    kmaj = kmaj.replace("sw128_offset(r, (k & 31) >> 2)", "(r * 128 + ((((k & 31) >> 2) ^ (r & 7)) << 4))")
    kPx = 32
    kGkChunk = kPx * 128

    def byte_k(px, ch):      # K-major, SWIZZLE_128B: rows = pixel, 32-channel chunks kGkChunk apart
        return (ch // 32) * kGkChunk + px * 128 + ((((ch % 32) // 4) ^ (px % 8)) * 16) + (ch % 4) * 4

    def byte_mn(px, c):      # MN-major, SWIZZLE_128B with a 32-byte base (UMMA layout type 1): LBO = chunk, SBO = 512 B per 4 pixels
        return (c // 32) * kGkChunk + (px // 4) * 512 + (px % 4) * 128 + ((((c % 32) // 8) ^ (px % 4)) * 32) + (c % 8) * 4

    seen_k, seen_mn = set(), set()
    for warp in range(8):                       # every warp converts the same pieces of G and of X
        for lane in range(32):
            c16, pxl = lane & 7, lane >> 3
            jc, p0 = warp & 3, (warp >> 2) * 4 + pxl
            ch = jc * 32 + c16 * 4
            env = dict(jc=jc, p0=p0, c16=c16, pxl=pxl, kGkChunk=kGkChunk)
            ko, mo = eval(k_off, {}, env), eval(mn_off, {}, env)
            for e in range(kPx // 8):
                px = p0 + 8 * e
                for i in range(4):              # the four channels of the 16-byte piece are contiguous in both images
                    assert ko + e * 1024 + 4 * i == byte_k(px, ch + i), (warp, lane, e, i)
                    assert mo + e * 1024 + 4 * i == byte_mn(px, ch + i), (warp, lane, e, i)
                seen_k.add(ko + e * 1024); seen_mn.add(mo + e * 1024)
    assert seen_k == set(range(0, 4 * kGkChunk, 16)) and seen_mn == set(range(0, 4 * kGkChunk, 16))      # each image tiled exactly once

    for px in range(kPx):                       # fragment / epilogue reads: element (px, c) of either image
        for c in range(128):
            assert eval(kmaj, {}, dict(r=px, k=c, kGkChunk=kGkChunk)) == byte_k(px, c), (px, c)
            assert eval(mnmaj, {}, dict(k=px, mn=c, kGkChunk=kGkChunk)) == byte_mn(px, c), (px, c)


def test_tc_fwd_piece_addresses_are_the_umma_image():
    """mlp_tc.cu, forward layer: converter thread (warp w, lane) owns chunk c = w & 3, rows r0 + 8 i; its piece address
    `c * kTChunk + sw128_offset(r0, u) + i * 1024` (lifted) must be the K-major 128-byte-swizzle address of (row, channel) in a 64-row
    tile, and the 256 threads x 8 pieces must tile the 32 KB stage exactly once."""
    src = open(os.path.join(ROOT, "gaussianavatar_b200", "csrc", "mlp_tc.cu")).read()
    tcc = open(os.path.join(ROOT, "gaussianavatar_b200", "csrc", "tc_common.cuh")).read()
    soff = _c_expr(src, r"const uint32_t soff = (.*?);\s")
    sw = re.search(r"uint32_t sw128_offset\(int r, int u\) \{ return (.*?); \}", tcc)
    assert sw
    sw_expr = re.sub(r"(\d+)u\b", r"\1", re.sub(r"\(uint32_t\)", "", sw.group(1)))
    sw128_offset = lambda r, u: eval(sw_expr, {}, dict(r=r, u=u))
    kTPx = 64
    kTChunk = kTPx * 128
    seen = set()
    for warp in range(8):
        for lane in range(32):
            rl, u = lane >> 3, lane & 7
            c, r0 = warp & 3, (warp >> 2) * 4 + rl
            base = eval(soff, {"sw128_offset": sw128_offset}, dict(c=c, r0=r0, u=u, kTChunk=kTChunk))
            for i in range(8):
                row, ch = r0 + 8 * i, c * 32 + u * 4
                want = (ch // 32) * kTChunk + row * 128 + ((((ch % 32) // 4) ^ (row % 8)) * 16)
                assert base + i * 1024 == want, (warp, lane, i)
                seen.add(base + i * 1024)
    assert seen == set(range(0, 4 * kTChunk, 16))
