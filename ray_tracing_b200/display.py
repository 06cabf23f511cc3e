"""RayTraceDisplay — mirror of the reference's display component (Assets/Scripts/Tracer/RayTraceDisplay.cs:9-23 +
Display.shader:42-47) and of its screenshot key (RayComputeManager.cs:106-111): the accumulated image divided by the
frame counter, shown / saved as an 8-bit sRGB picture.  The division and encoding run on the GPU (rtDisplay)."""
from __future__ import annotations

import struct
import zlib

import numpy as np


class RayTraceDisplay:
    def __init__(self, raytracer):
        self.raytracer = raytracer                      # a RayComputeManager

    def OnRenderImage(self) -> np.ndarray:
        """(H, W, 4) uint8, top row first (screen order).  Frame = numAccumulatedFrames when accumulating, else 1 —
        including the reference's off-by-one: the counter is one ahead of the number of summed frames (SURVEY §3.4)."""
        m = self.raytracer
        acc = bool(m.accumulate)
        img = m.context.display(acc, m.numAccumulatedFrames if acc else 1)
        return img[::-1]

    def save_screenshot(self, path: str) -> None:
        write_png(path, self.OnRenderImage()[..., :3])

    def DenoisedImage(self) -> np.ndarray:
        """The image the last Denoise() of the manager wrote (rtDisplayDenoised), (H, W, 4) uint8, top row first."""
        return self.raytracer.context.display_denoised()[::-1]

    def save_denoised(self, path: str) -> None:
        write_png(path, self.DenoisedImage()[..., :3])

    def MeanImage(self) -> np.ndarray:
        """The per-pixel mean of the accumulated image (rtDisplayMean): what an adaptively sampled render (RenderFrameAdaptive), whose
        pixels have different frame counts, looks like.  (H, W, 4) uint8, top row first."""
        return self.raytracer.display_mean()[::-1]

    def save_mean(self, path: str) -> None:
        write_png(path, self.MeanImage()[..., :3])

    def DebugView(self, visMode: int, debugVisScale: float) -> np.ndarray:
        """The reference's debug view (visMode / debugVisScale, RayCommon.hlsl:24-26): heat map of the per-pixel traversal counters
        of the counting launches, (H, W, 4) uint8, top row first.  See RayComputeManager.debug_view."""
        return self.raytracer.debug_view(visMode, debugVisScale)[::-1]

    def save_debug_view(self, path: str, visMode: int, debugVisScale: float) -> None:
        write_png(path, self.DebugView(visMode, debugVisScale)[..., :3])


def write_png(path: str, rgb8: np.ndarray) -> None:
    h, w, _ = rgb8.shape
    raw = b"".join(b"\x00" + np.ascontiguousarray(rgb8[y]).tobytes() for y in range(h))

    def chunk(tag: bytes, data: bytes) -> bytes:
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
                + chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def write_exr(path: str, rgba: np.ndarray) -> None:
    """The float4 render target as an OpenEXR file (single part, scan lines, no compression, four FLOAT channels) — the lossless
    way out for AccumulatedRender / FrameRender (the reference's only exporter is the 8-bit PNG screenshot, RayComputeManager.cs:106-111).
    Rows are written top to bottom as EXR wants them; pass the image already in display orientation (row 0 = top)."""
    img = np.ascontiguousarray(rgba, dtype=np.float32)
    if img.ndim != 3 or img.shape[2] != 4:
        raise ValueError("write_exr expects an (H, W, 4) float image")
    h, w, _ = img.shape

    def attr(name: str, typ: str, data: bytes) -> bytes:
        return name.encode() + b"\x00" + typ.encode() + b"\x00" + struct.pack("<i", len(data)) + data

    chlist = b"".join(c + b"\x00" + struct.pack("<iBxxxii", 2, 0, 1, 1) for c in (b"A", b"B", b"G", b"R")) + b"\x00"     # FLOAT = 2, alphabetical
    box = struct.pack("<iiii", 0, 0, w - 1, h - 1)
    header = (attr("channels", "chlist", chlist) + attr("compression", "compression", b"\x00") + attr("dataWindow", "box2i", box)
              + attr("displayWindow", "box2i", box) + attr("lineOrder", "lineOrder", b"\x00") + attr("pixelAspectRatio", "float", struct.pack("<f", 1.0))
              + attr("screenWindowCenter", "v2f", struct.pack("<ff", 0.0, 0.0)) + attr("screenWindowWidth", "float", struct.pack("<f", 1.0)) + b"\x00")
    magic = struct.pack("<iI", 20000630, 2)
    row_bytes = 4 * w * 4
    table_pos = len(magic) + len(header)
    first = table_pos + 8 * h
    offsets = struct.pack(f"<{h}Q", *(first + y * (8 + row_bytes) for y in range(h)))
    with open(path, "wb") as f:
        f.write(magic + header + offsets)
        for y in range(h):
            row = img[y]
            f.write(struct.pack("<ii", y, row_bytes) + row[:, 3].tobytes() + row[:, 2].tobytes() + row[:, 1].tobytes() + row[:, 0].tobytes())


def write_cubemap_exr(path: str, faces: np.ndarray) -> None:
    """One probe of rtBakeCubemaps as an OpenEXR horizontal strip, 6N wide and N high: the faces left to right in their order (+X, -X,
    +Y, -Y, +Z, -Z), each with row 0 at the top, rgb and alpha 1.  `faces` is one probe's (6, N, N) CUBE_TEXEL_DTYPE records or a
    (6, N, N, 3) float array."""
    rgb = np.asarray(faces["rgb"] if getattr(faces, "dtype", None) is not None and faces.dtype.names else faces, dtype=np.float32)
    if rgb.ndim != 4 or rgb.shape[0] != 6 or rgb.shape[1] != rgb.shape[2] or rgb.shape[3] != 3:
        raise ValueError("write_cubemap_exr expects one probe's (6, N, N) texels or a (6, N, N, 3) float array")
    n = rgb.shape[1]
    strip = np.ones((n, 6 * n, 4), dtype=np.float32)
    strip[:, :, :3] = rgb.transpose(1, 0, 2, 3).reshape(n, 6 * n, 3)
    write_exr(path, strip)


def read_exr(path: str) -> np.ndarray:
    """Reads back what write_exr wrote (uncompressed scan lines, FLOAT channels A, B, G, R) -> (H, W, 4) float32 RGBA."""
    data = open(path, "rb").read()
    if struct.unpack_from("<i", data, 0)[0] != 20000630:
        raise ValueError("not an OpenEXR file")
    off, attrs = 8, {}
    while data[off] != 0:
        end = data.index(b"\x00", off); name = data[off:end].decode(); off = end + 1
        end = data.index(b"\x00", off); off = end + 1
        size = struct.unpack_from("<i", data, off)[0]; off += 4
        attrs[name] = data[off:off + size]; off += size
    off += 1
    if attrs["compression"] != b"\x00":
        raise ValueError("only uncompressed EXR files are read")
    x0, y0, x1, y1 = struct.unpack("<iiii", attrs["dataWindow"])
    w, h = x1 - x0 + 1, y1 - y0 + 1
    offsets = struct.unpack_from(f"<{h}Q", data, off)
    out = np.empty((h, w, 4), dtype=np.float32)
    for o in offsets:
        y, n = struct.unpack_from("<ii", data, o)
        chans = np.frombuffer(data, dtype="<f4", count=4 * w, offset=o + 8).reshape(4, w)       # A, B, G, R
        out[y - y0] = chans[::-1].T
    return out
