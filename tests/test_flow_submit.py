"""KITTI-2015 flow submission without a GPU: the oracle against the outputs frozen from the reference's own flowlib,
flow_io and compute_err; the kernels compiled by g++ against the CPU execution-model simulator (tests/sim) against
fixture, oracle and torch's CPU interpolate; the PNG codec against OpenCV.  The same cases run on the H100 in
tests/test_gpu_flow_submit.py."""
import os
import numpy as np
import pytest
import torch
from cc_b200.flowutils import flow_io
from oracle import flow_submit as OF
from tests import flow_submit_cases as SC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


def test_oracle_equals_reference():
    d = SC.g()
    for name, (h, w, Hg, Wg) in SC.SUBMIT.items():
        mask, cam, fwd, total = OF.submit_flows(*(torch.from_numpy(d[name + k]) for k in ('_emask', '_cam', '_fwd')), Hg, Wg, 0.01)
        assert np.array_equal(mask[0].numpy(), d[name + '_mask'])
        assert np.array_equal(OF.kitti_png_rows(total[0, 0].numpy(), total[0, 1].numpy()), d[name + '_png'])
        import hashlib
        assert hashlib.sha256(OF.flo_bytes(total[0, 0].numpy(), total[0, 1].numpy())).hexdigest() == str(d[name + '_flo_sha256'])
        viz = OF.flow_to_image(np.hstack((cam[0].numpy(), fwd[0].numpy(), total[0].numpy())))
        assert np.array_equal(viz, d[name + '_viz'] / 255.)
    wrap = d['wrap_flow']
    assert np.array_equal(OF.kitti_png_rows(wrap[0], wrap[1]), d['wrap_png'])
    assert OF.flo_bytes(wrap[0], wrap[1]) == d['wrap_flo'].tobytes()
    for name in SC.COLOR:
        flow = d[name + '_flow']
        assert np.array_equal(OF.flow_to_image(np.hstack(list(flow)) if flow.ndim == 4 else flow), d[name + '_viz'] / 255.), name
    assert np.array_equal(OF.make_color_wheel(), d['wheel'])
    u, v, valid = OF.decode_png_rows(d['err_gt'])
    up, vp, _ = OF.decode_png_rows(d['err_pred'])
    assert np.array_equal(np.stack([u[0], v[0], valid[0], up[0], vp[0]]), d['err_decoded_row0'])
    assert OF.compute_err(u, v, valid, up, vp)[0] == d['err_out'].tolist()


def test_flow_io_matches_reference(tmp_path):
    """flow_write_png / flow_read_png / flow_write on numpy arrays and tensors: the reference's rows, decoding and bytes."""
    d = SC.g()
    wrap = d['wrap_flow']
    for u, v in ((wrap[0], wrap[1]), (torch.from_numpy(wrap[0]), torch.from_numpy(wrap[1]))):
        flow_io.flow_write_png(str(tmp_path / 'a_10.png'), u=u, v=v)
        assert np.array_equal(flow_io.read_png(str(tmp_path / 'a_10.png')), d['wrap_png'])
        flow_io.flow_write(str(tmp_path / 'a_10.flo'), u, v)
        assert (tmp_path / 'a_10.flo').read_bytes() == d['wrap_flo'].tobytes()
    flow_io.flow_write(str(tmp_path / 'b.flo'), wrap)
    assert (tmp_path / 'b.flo').read_bytes() == d['wrap_flo'].tobytes()
    flow_io.write_png(str(tmp_path / 'gt.png'), d['err_gt'])
    u, v, valid = flow_io.flow_read_png(str(tmp_path / 'gt.png'))
    assert np.array_equal(np.stack([u[0], v[0], valid[0]]), d['err_decoded_row0'][:3]) and valid.dtype == np.uint16


def test_png_codec_against_opencv(tmp_path):
    """Files of the writer decode identically with OpenCV (BGR order), and the decoder reads OpenCV's filtered PNGs
    (libpng picks Sub / Up / Average / Paeth per row) at 16 and 8 bits."""
    cv2 = pytest.importorskip('cv2')
    rs = np.random.RandomState(3)
    smooth = (np.cumsum(np.cumsum(rs.randint(-300, 300, size=(37, 53, 3)), 0), 1) % 65536).astype(np.uint16)
    seen = set()
    for img in (SC.g()['err_gt'], SC.g()['small_png'], smooth, (smooth >> 8).astype(np.uint8)):
        p = str(tmp_path / 'w.png')
        flow_io.write_png(p, img)
        back = cv2.imread(p, cv2.IMREAD_UNCHANGED)
        assert back.dtype == img.dtype and np.array_equal(back[:, :, ::-1], img)
        for flt in ('NONE', 'SUB', 'UP', 'AVG', 'PAETH', 'ALL_FILTERS'):
            q = str(tmp_path / ('cv_%s.png' % flt))
            assert cv2.imwrite(q, np.ascontiguousarray(img[:, :, ::-1]), [cv2.IMWRITE_PNG_FILTER, getattr(cv2, 'IMWRITE_PNG_' + flt
                                                                                                         if flt == 'ALL_FILTERS' else 'IMWRITE_PNG_FILTER_' + flt)])
            assert np.array_equal(flow_io.read_png(q), img), flt
            with open(q, 'rb') as f:
                seen |= _filter_types(f.read(), img.shape[0])
    assert seen == {0, 1, 2, 3, 4}, 'OpenCV wrote filter types %s only' % seen
    gray = (smooth[:, :, 0] >> 3).astype(np.uint16)
    assert cv2.imwrite(str(tmp_path / 'g.png'), gray)
    assert np.array_equal(flow_io.read_png(str(tmp_path / 'g.png'))[:, :, 0], gray)


def _filter_types(data, h):
    import struct
    import zlib
    pos, idat = 8, []
    while pos < len(data):
        n, kind = struct.unpack('>I4s', data[pos:pos + 8])
        if kind == b'IDAT':
            idat.append(data[pos + 8:pos + 8 + n])
        pos += 12 + n
    return set(np.frombuffer(zlib.decompress(b''.join(idat)), np.uint8).reshape(h, -1)[:, 0].tolist())


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('case', SC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(CPU)


@pytest.mark.usefixtures('sim_lib')
def test_kitti_size_sample():
    """256x832 -> 375x1242 through the simulator: the KITTI triplet, .flo payload and full flows against the oracle."""
    SC.case_random_submit(CPU, B=1, sizes=SC.KITTI, seed=11, colors=False)
