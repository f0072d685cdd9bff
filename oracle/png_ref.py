"""CPU restatement of the PNG files the device encoder (ops.mask_png, fb200_mask_png) writes, with the standard library only.

TEST INFRASTRUCTURE - NOT PRODUCT CODE.  The format is what `cv2.imencode(".png", crop * 255)` writes for a 0/255 crop: SUB-filtered rows (NONE for a
one-pixel-wide image), zlib's deflate with strategy Z_RLE and memLevel 8, a CMF with the smallest window >= 256 bytes covering the filtered bytes (at most
32 KiB), 8192-byte IDAT chunks."""
import struct
import zlib

import numpy as np
import torch


def png_file(m) -> bytes:
    """the PNG file cv2.imencode(".png", m) writes for a 2-D uint8 array m of 0 / 255"""
    h, w = m.shape
    f = np.empty((h, w + 1), np.uint8)
    f[:, 0] = 1 if w > 1 else 0  # SUB; libpng filters a one-pixel-wide image with NONE
    f[:, 1:] = np.diff(m.astype(np.int16), axis=1, prepend=0).astype(np.uint8)
    data = f.tobytes()
    c = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
    z = bytearray(c.compress(data) + c.flush())
    cinfo = 0
    while cinfo < 7 and len(data) > 256 << cinfo:
        cinfo += 1
    z[0] = cinfo << 4 | 8
    z[1] = 31 - (z[0] << 8) % 31

    def chunk(kind, payload):
        return struct.pack(">I", len(payload)) + kind + payload + struct.pack(">I", zlib.crc32(kind + payload))

    idat = b"".join(chunk(b"IDAT", bytes(z[k:k + 8192])) for k in range(0, len(z), 8192))
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) + idat + chunk(b"IEND", b"")


def mask_png(masks, bbox):
    """ops.mask_png on the CPU: masks [n,H,W] (non-zero = set), bbox [n,4] xyxy -> (bytes uint8 [sum(lengths)], lengths int32 [n]), crop i being
    masks[i][y1:min(y2,H), x1:min(x2,W)] and an empty crop a length of 0"""
    H, W = masks.shape[1:]
    files = []
    for i in range(masks.shape[0]):
        x1, y1, x2, y2 = (int(v) for v in bbox[i])
        crop = (torch.as_tensor(masks[i, y1:min(y2, H), x1:min(x2, W)]) != 0).to(torch.uint8) * 255
        files.append(png_file(crop.numpy()) if crop.numel() else b"")
    lengths = torch.tensor([len(f) for f in files], dtype=torch.int32)
    return torch.frombuffer(bytearray(b"".join(files) or b"\0"), dtype=torch.uint8)[:int(lengths.sum())], lengths
