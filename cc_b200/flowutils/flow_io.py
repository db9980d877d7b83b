"""The reference's flowutils/flow_io.py entry points for KITTI and Middlebury flow files, without pypng: 16-bit PNGs are
written and read by the codec below (zlib and struct only).

  flow_write_png(fpath, u, v, valid=None)   KITTI flow PNG: uint16 RGB (u*64 + 2^15, v*64 + 2^15, valid), the encoding in
                                            fp64 with numpy's float64 -> uint16 cast (flows past +-512 px wrap)
  flow_read_png(fpath) -> u, v, valid       its decoding: (x - 2^15) / 64 in fp64, valid as uint16
  flow_write(filename, uv, v=None)          Middlebury .flo: 'PIEH', int32 width, int32 height, u, v interleaved as fp32

u, v (and uv) may be numpy arrays or tensors on any device.  The device path of a whole submission is
cc_b200.evaluate.flow_submission, whose uint16 triplet and .flo payload these writers store (write_png, write_flo_payload).
"""
import struct
import zlib
import numpy as np

_SIGNATURE = b'\x89PNG\r\n\x1a\n'
_CHANNELS = {0: 1, 2: 3, 4: 2, 6: 4}          # colour type -> samples per pixel (grey, RGB, grey+alpha, RGBA)


def _host(a):
    return a.detach().cpu().numpy() if hasattr(a, 'detach') else np.asarray(a)


def _chunk(kind, data):
    return struct.pack('>I', len(data)) + kind + data + struct.pack('>I', zlib.crc32(kind + data) & 0xffffffff)


def encode_png(img):
    """PNG bytes of a uint8 or uint16 image [H, W] or [H, W, C] (C = 1, 2, 3, 4), every row with filter type 0."""
    img = np.asarray(img)
    if img.ndim == 2:
        img = img[:, :, None]
    h, w, c = img.shape
    depth = {np.dtype(np.uint8): 8, np.dtype(np.uint16): 16}[img.dtype]
    ctype = {1: 0, 2: 4, 3: 2, 4: 6}[c]
    raw = np.ascontiguousarray(img.astype('>u2' if depth == 16 else np.uint8)).view(np.uint8).reshape(h, -1)
    rows = np.concatenate([np.zeros((h, 1), np.uint8), raw], axis=1)
    return _SIGNATURE + _chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, depth, ctype, 0, 0, 0)) + \
        _chunk(b'IDAT', zlib.compress(rows.tobytes(), 6)) + _chunk(b'IEND', b'')


def write_png(fpath, img):
    with open(fpath, 'wb') as f:
        f.write(encode_png(img))


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def _unfilter(data, h, stride, bpp):
    """The scanlines of a non-interlaced image from the decompressed stream: each row's filter byte (0 None, 1 Sub, 2 Up,
    3 Average, 4 Paeth) undone against the row above and the byte `bpp` to the left."""
    buf = np.frombuffer(data, np.uint8)
    if buf.size != h * (stride + 1):
        raise ValueError('PNG: %d bytes of image data, %d expected' % (buf.size, h * (stride + 1)))
    rows = buf.reshape(h, stride + 1)
    out = np.zeros((h, stride), np.uint8)
    prior = np.zeros(stride, np.int32)
    for y in range(h):
        kind, f = rows[y, 0], rows[y, 1:].astype(np.int32)
        if kind == 0:
            cur = f
        elif kind == 2:
            cur = (f + prior) & 0xff
        elif kind == 1:                      # Sub: a running sum along each of the bpp interleaved byte lanes
            cur = np.cumsum(f.reshape(-1, bpp), axis=0).reshape(-1) & 0xff
        elif kind in (3, 4):                 # Average / Paeth depend on the reconstructed left pixel: one pixel at a time
            cur = np.zeros(stride, np.int32)
            left, up_left = np.zeros(bpp, np.int32), np.zeros(bpp, np.int32)
            for x in range(0, stride, bpp):
                up = prior[x:x + bpp]
                pred = (left + up) >> 1 if kind == 3 else _paeth(left, up, up_left)
                left = (f[x:x + bpp] + pred) & 0xff
                cur[x:x + bpp] = left
                up_left = up
        else:
            raise ValueError('PNG: unknown filter type %d' % kind)
        out[y] = cur
        prior = cur
    return out


def decode_png(data):
    """A non-interlaced, non-palette 8- or 16-bit PNG -> uint8 / uint16 array [H, W, C]."""
    if data[:8] != _SIGNATURE:
        raise ValueError('PNG: bad signature')
    pos, idat, hdr = 8, [], None
    while pos < len(data):
        n, kind = struct.unpack('>I4s', data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        if kind == b'IHDR':
            hdr = struct.unpack('>IIBBBBB', body)
        elif kind == b'IDAT':
            idat.append(body)
        elif kind == b'IEND':
            break
        pos += 12 + n
    if hdr is None:
        raise ValueError('PNG: no IHDR chunk')
    w, h, depth, ctype, _, _, interlace = hdr
    if ctype not in _CHANNELS or depth not in (8, 16) or interlace != 0:
        raise ValueError('PNG: colour type %d, bit depth %d, interlace %d is not supported' % (ctype, depth, interlace))
    c = _CHANNELS[ctype]
    bpp = c * depth // 8
    rows = _unfilter(zlib.decompress(b''.join(idat)), h, w * bpp, bpp)
    if depth == 16:
        return rows.view('>u2').astype(np.uint16).reshape(h, w, c)
    return rows.reshape(h, w, c)


def read_png(fpath):
    with open(fpath, 'rb') as f:
        return decode_png(f.read())


def kitti_encode(u, v, valid=None):
    """flow_write_png's image: uint16 [H, W, 3]."""
    u, v = _host(u), _host(v)
    valid_ = np.ones(u.shape, dtype='uint16') if valid is None else _host(valid).astype('uint16')
    with np.errstate(invalid='ignore'):
        return np.dstack((((u.astype('float64') * 64.0) + 2 ** 15).astype('uint16'),
                          ((v.astype('float64') * 64.0) + 2 ** 15).astype('uint16'), valid_))


def flow_write_png(fpath, u, v, valid=None):
    """Write KITTI optical flow (flow_io.py:120-150)."""
    write_png(fpath, kitti_encode(u, v, valid))


def flow_read_png(fpath):
    """Read KITTI optical flow (flow_io.py:96-117): u, v in float64 pixels and the valid channel (uint16)."""
    img = read_png(fpath)
    return (img[:, :, 0].astype('float64') - 2 ** 15) / 64.0, (img[:, :, 1].astype('float64') - 2 ** 15) / 64.0, img[:, :, 2]


def write_flo_payload(filename, uv_hw2):
    """A .flo file of an fp32 [H, W, 2] array (u, v interleaved), as flow_write writes it."""
    uv = np.ascontiguousarray(_host(uv_hw2), dtype=np.float32)
    h, w, _ = uv.shape
    with open(filename, 'wb') as f:
        f.write(b'PIEH' + np.array([w, h], np.int32).tobytes() + uv.tobytes())


def flow_write(filename, uv, v=None):
    """Write optical flow in the Middlebury .flo format (flow_io.py:57-93): uv [2,H,W] or [H,W,2], or u and v."""
    if v is None:
        uv = _host(uv)
        assert uv.ndim == 3
        if uv.shape[0] == 2:
            u, v = uv[0], uv[1]
        elif uv.shape[2] == 2:
            u, v = uv[:, :, 0], uv[:, :, 1]
        else:
            raise ValueError('Wrong format for flow input')
    else:
        u, v = _host(uv), _host(v)
    assert u.shape == v.shape
    write_flo_payload(filename, np.stack([np.asarray(u, np.float64), np.asarray(v, np.float64)], -1).astype(np.float32))
