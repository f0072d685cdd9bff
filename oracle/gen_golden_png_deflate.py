"""Golden PNG files of mask crops for the device PNG encoder (fb200_mask_png): `cv2.imencode(".png", crop * 255)` of seeded crops -> tests/golden/png_deflate.npz.
Needs OpenCV:  python -m oracle.gen_golden_png_deflate

The cases cover crops from 1x1 to 1080x1920; all-zero, all-one, noise, discs, single rows and columns (a one-pixel-wide image is filtered with NONE, not SUB);
column stripes (every filtered byte a literal); runs longer than 258; filtered sizes just below, at and above every CINFO window boundary (256 ... 16384, 32768);
streams of several deflate blocks (one whose symbol count is exactly 16383, which zlib follows with an empty last block) and of several IDAT chunks.
Each stream's deflate block headers are parsed: the fixture must hold fixed and dynamic blocks.  Stored blocks are searched for on every mask of at most 12 pixels
and on seeded random small masks; none has been found, and the count of masks searched is recorded in the fixture's `stored_search`."""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "png_deflate.npz")


def _bits(data: bytes):
    for byte in data:
        for k in range(8):
            yield (byte >> k) & 1


class _Reader:
    def __init__(self, data: bytes):
        self.it, self.pos = _bits(data), 0

    def get(self, n: int) -> int:
        v = 0
        for k in range(n):
            v |= next(self.it) << k
        self.pos += n
        return v

    def sym(self, table) -> int:
        code = length = 0
        while (length, code) not in table:
            code, length = code << 1 | self.get(1), length + 1
        return table[(length, code)]


def _canonical(lengths):
    count = [0] * 16
    for n in lengths:
        count[n] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    table = {}
    for s, n in enumerate(lengths):
        if n:
            table[(n, nxt[n])] = s
            nxt[n] += 1
    return table


_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0] * 8 + [1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
_DEXT = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


def block_types(zstream: bytes):
    """BTYPE of every deflate block of a zlib stream (0 stored, 1 fixed, 2 dynamic)"""
    r, types = _Reader(zstream[2:-4]), []
    while True:
        final, kind = r.get(1), r.get(2)
        types.append(kind)
        if kind == 0:
            r.get((8 - r.pos % 8) % 8)
            n = r.get(16)
            r.get(16 + 8 * n)
        else:
            if kind == 1:
                lt = _canonical([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
                dt = _canonical([5] * 30)
            else:
                hlit, hdist, hclen = r.get(5) + 257, r.get(5) + 1, r.get(4) + 4
                order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
                cl = [0] * 19
                for k in range(hclen):
                    cl[order[k]] = r.get(3)
                ct, lens = _canonical(cl), []
                while len(lens) < hlit + hdist:
                    s = r.sym(ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + r.get(2))
                    elif s == 17:
                        lens += [0] * (3 + r.get(3))
                    else:
                        lens += [0] * (11 + r.get(7))
                lt, dt = _canonical(lens[:hlit]), _canonical(lens[hlit:])
            while True:
                s = r.sym(lt)
                if s == 256:
                    break
                if s > 256:
                    r.get(_LEXT[s - 257])
                    r.get(_DEXT[r.sym(dt)])
        if final:
            return types


def zlib_stream(png: bytes) -> bytes:
    i, z = 8, b""
    while i < len(png):
        n = int.from_bytes(png[i:i + 4], "big")
        if png[i + 4:i + 8] == b"IDAT":
            z += png[i + 8:i + 8 + n]
        i += 12 + n
    return z


def cases():
    rng = np.random.default_rng(11)
    out = {"one_1x1": np.ones((1, 1), bool), "zero_1x1": np.zeros((1, 1), bool), "zero_64x64": np.zeros((64, 64), bool),
           "one_200x300": np.ones((200, 300), bool), "noise_300x400": rng.random((300, 400)) > 0.5, "sparse_noise_240x320": rng.random((240, 320)) > 0.97,
           "row_1x700": rng.random((1, 700)) > 0.4, "column_500x1": rng.random((500, 1)) > 0.5, "zero_column_400x1": np.zeros((400, 1), bool),
           "stripes_127x128": np.tile(np.arange(128) % 2 == 0, (127, 1)), "stripes_64x1000": np.tile(np.arange(1000) % 2 == 1, (64, 1))}
    yy, xx = np.mgrid[:1080, :1920]
    out["disc_1080x1920"] = np.hypot(yy - 500, xx - 900) < 450
    yy, xx = np.mgrid[:333, :517]
    out["discs_333x517"] = (np.hypot(yy - 120, xx - 200) < 90) | (np.hypot(yy - 250, xx - 400) < 70)
    runs = np.ones((5, 1000), bool)
    runs[1, 259] = runs[2, 261] = runs[3, 516] = runs[4, 519] = False
    out["runs_5x1000"] = runs
    for N in (256, 512, 1024, 2048, 4096, 8192, 16384, 32768):
        for d in (-1, 0, 1):
            n = N + d
            w1 = max(k for k in range(1, int(n ** 0.5) + 1) if n % k == 0)  # h * (w + 1) == n with w + 1 the largest divisor <= sqrt(n)
            w1 = w1 if w1 >= 2 else n
            out[f"window_{n}_{n // w1}x{w1 - 1}"] = rng.random((n // w1, w1 - 1)) > 0.5
    return out


def main():
    import cv2

    names, shapes, bits, pngs, kinds = [], [], [], [], []
    for name, m in cases().items():
        png = cv2.imencode(".png", m.astype(np.uint8) * 255)[1].tobytes()
        names.append(name)
        shapes.append(m.shape)
        bits.append(np.packbits(m.ravel()))
        pngs.append(np.frombuffer(png, np.uint8))
        kinds.append(block_types(zlib_stream(png)))
    flat = [k for t in kinds for k in t]
    assert 1 in flat and 2 in flat, "the fixture needs fixed and dynamic blocks"
    assert max(len(t) for t in kinds) >= 4 and any(len(p) > 3 * 8192 for p in pngs)
    searched = stored = 0
    for h in range(1, 13):
        for w in range(1, 13 // h + 1):
            for v in range(2 ** (h * w)):
                m = (np.array([(v >> k) & 1 for k in range(h * w)], np.uint8).reshape(h, w)) * 255
                stored += 0 in block_types(zlib_stream(cv2.imencode(".png", m)[1].tobytes()))
                searched += 1
    rng = np.random.default_rng(12)
    for _ in range(5000):
        h, w = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        m = ((rng.random((h, w)) > rng.random()) if rng.random() < 0.7 else np.tile(np.arange(w) % 2 == 0, (h, 1))).astype(np.uint8) * 255
        stored += 0 in block_types(zlib_stream(cv2.imencode(".png", m)[1].tobytes()))
        searched += 1
    assert stored == 0, f"{stored} masks produced a stored block"
    offs = np.cumsum([0] + [len(b) for b in bits])
    poffs = np.cumsum([0] + [len(p) for p in pngs])
    np.savez_compressed(PATH, names=np.array(names), shapes=np.array(shapes, np.int32), bits=np.concatenate(bits), bit_offsets=offs, png=np.concatenate(pngs),
                        png_offsets=poffs, block_types=np.array([",".join(map(str, t)) for t in kinds]),
                        stored_search=np.array(f"0 stored blocks in {searched} masks (every mask of at most 12 pixels, 5000 seeded random / stripe masks up to 39x39)"),
                        cv2=np.array(cv2.__version__))
    print("wrote", PATH, len(names), "cases, block types", sorted(set(flat)), "largest block count", max(len(t) for t in kinds))


def load(path=PATH):
    """-> list of (name, bool crop, PNG bytes)"""
    g = np.load(path)
    out = []
    for k, name in enumerate(g["names"]):
        h, w = (int(v) for v in g["shapes"][k])
        m = np.unpackbits(g["bits"][g["bit_offsets"][k]:g["bit_offsets"][k + 1]])[:h * w].reshape(h, w).astype(bool)
        out.append((str(name), m, g["png"][g["png_offsets"][k]:g["png_offsets"][k + 1]].tobytes()))
    return out


if __name__ == "__main__":
    main()
