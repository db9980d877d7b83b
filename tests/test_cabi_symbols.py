"""The C-ABI library loads and exports every symbol include/*.h declares (no compute calls), and the Python binding
declares every prototype and descriptor struct exactly as the headers do."""
import ctypes
import itertools
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_source():
    src = ''.join(open(os.path.join(ROOT, 'include', f)).read() for f in sorted(os.listdir(os.path.join(ROOT, 'include')))
                  if f.endswith('.h'))
    return re.sub(r'/\*.*?\*/', '', src, flags=re.S)


def _ctype(tokens):
    """C type spelled as the binding's table spells it: 'const float*', 'float* const*', 'unsigned long long*' ..."""
    out = ''
    for t in tokens:
        out += t if t == '*' else (' ' if out else '') + t
    return out


def declared():
    return sorted(set(re.findall(r'\b(ccb_[a-z0-9_]+)\s*\(', _header_source())))


def header_prototypes():
    """{name: (return type, [parameter types])} of every prototype of include/*.h."""
    src = re.sub(r'^\s*#.*$', '', _header_source(), flags=re.M)
    protos = {}
    for m in re.finditer(r'([^;{}]*?)\b(ccb_\w+)\s*\(([^()]*)\)\s*;', src):
        params = [p for p in m.group(3).split(',') if p.strip() not in ('', 'void')]
        protos[m.group(2)] = (_ctype(re.findall(r'\w+|\*', m.group(1))),
                              [_ctype(re.findall(r'\w+|\*', p)[:-1]) for p in params])      # [:-1]: the parameter name
    return protos


def header_structs():
    """{struct name: [(field, C type, array extents)]} of every typedef struct of include/*.h."""
    src = _header_source()
    macros = {k: int(v) for k, v in re.findall(r'#define\s+(\w+)\s+(\d+)', src)}
    structs = {}
    for name, body in re.findall(r'typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*\w+\s*;', src, flags=re.S):
        fields = []
        for decl in body.split(';'):
            if not decl.strip():
                continue
            first, *rest = decl.split(',')
            m = re.match(r'\s*(.*?)\s*(\w+)\s*((?:\[\s*\w+\s*\])*)\s*$', first, flags=re.S)
            ctype, base = _ctype(re.findall(r'\w+|\*', m.group(1))), m.group(1).replace('*', '').strip()
            decls = [(ctype, m.group(2), m.group(3))]
            for r in rest:              # further declarators of the same line: the base type plus their own stars
                m = re.match(r'\s*(\**)\s*(\w+)\s*((?:\[\s*\w+\s*\])*)\s*$', r)
                decls.append((_ctype(re.findall(r'\w+|\*', base) + list(m.group(1))), m.group(2), m.group(3)))
            for ctype, field, dims in decls:
                ext = tuple(macros[d] if d in macros else int(d) for d in re.findall(r'\[\s*(\w+)\s*\]', dims))
                fields.append((field, ctype, ext))
        structs[name] = fields
    return structs


def _struct_fields(cls):
    """[(field, C type as far as ctypes tells it, array extents)]; a pointer field is c_void_p: any 'T*'."""
    names = {ctypes.c_int: 'int', ctypes.c_longlong: 'long long', ctypes.c_float: 'float', ctypes.c_void_p: '*'}
    out = []
    for field, t in cls._fields_:
        ext = []
        while issubclass(t, ctypes.Array):
            ext.append(t._length_)
            t = t._type_
        out.append((field, names.get(t, t.__name__), tuple(ext)))
    return out


def binding_mismatches(sigs, structs):
    """Every difference between a signature table / descriptor Structures (as cc_b200._lib declares them) and the headers,
    one readable line each."""
    from cc_b200 import _lib
    protos, hstructs = header_prototypes(), header_structs()
    bad = ['%s: declared by the headers, not by the binding' % n for n in sorted(set(protos) - set(sigs))]
    bad += ['%s: in the binding, not declared by the headers' % n for n in sorted(set(sigs) - set(protos))]
    for name in sorted(set(protos) & set(sigs)):
        hret, hparams = protos[name]
        ret, params = sigs[name]
        params = [p for p in params.split(', ') if p]
        if ('int' if ret == _lib.STATUS else ret) != hret:
            bad.append('%s: returns %s, the binding says %s' % (name, hret, ret))
        if len(params) != len(hparams):
            bad.append('%s: %d parameters, the binding has %d' % (name, len(hparams), len(params)))
            continue
        for i, (h, p) in enumerate(zip(hparams, params)):
            marker, ctype = p.split(' ', 1) if p.split(' ')[0] in ('host', 'handle') else ('', p)
            if ctype != h or (marker == 'handle' and h != 'void*') or (marker == 'host' and not h.endswith('*')):
                bad.append('%s argument %d: %s, the binding says %s' % (name, i, h, p))
    for sname, fields in sorted(hstructs.items()):
        if sname not in structs:
            bad.append('struct %s: no ctypes Structure' % sname)
            continue
        want = [(f, '*' if t.endswith('*') else t, ext) for f, t, ext in fields]
        for i, (w, g) in enumerate(itertools.zip_longest(want, _struct_fields(structs[sname]))):
            if w != g:
                bad.append('struct %s field %d: header %s, ctypes %s' % (sname, i, w, g))
                break
    bad += ['struct %s: not declared by the headers' % s for s in sorted(set(structs) - set(hstructs))]
    return bad


def test_header_symbols_exported():
    import __graft_entry__ as ge
    path = ge.build()
    lib = ctypes.CDLL(path)
    names = declared()
    assert len(names) >= 20
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    lib.ccb_is_simulator.restype = ctypes.c_int
    assert lib.ccb_is_simulator() == 0
    lib.ccb_last_error_string.restype = ctypes.c_char_p
    assert lib.ccb_last_error_string() is not None


def test_binding_table_matches_headers():
    from cc_b200 import _lib
    assert sorted(_lib._SIGS) == declared()
    assert len(header_structs()) == 4
    assert binding_mismatches(_lib._SIGS, _lib.STRUCTS) == []


def test_binding_check_reports_planted_mismatches():
    """The comparison is not vacuous: a long long narrowed to int, a dropped parameter, a constness slip, a field type
    and a reordered struct are each reported."""
    import ctypes as C
    from cc_b200 import _lib
    sigs = dict(_lib._SIGS)
    ret, params = sigs['ccb_resize_u8']
    assert params.count('long long') == 1
    sigs['ccb_resize_u8'] = (ret, params.replace('long long', 'int'))
    assert binding_mismatches(sigs, _lib.STRUCTS) == ['ccb_resize_u8 argument 8: long long, the binding says int']
    sigs = dict(_lib._SIGS, ccb_upsample2x_fwd=(_lib.STATUS, 'const float*, float*, int, int, ccb_stream_t'))
    assert binding_mismatches(sigs, _lib.STRUCTS) == ['ccb_upsample2x_fwd: 6 parameters, the binding has 5']
    sigs = dict(_lib._SIGS, ccb_upsample2x_fwd=(_lib.STATUS, 'float*, float*, int, int, int, ccb_stream_t'))
    assert binding_mismatches(sigs, _lib.STRUCTS) == ['ccb_upsample2x_fwd argument 0: const float*, the binding says float*']
    sigs = dict(_lib._SIGS, ccb_launch_count=('int', ''))
    assert binding_mismatches(sigs, _lib.STRUCTS) == ['ccb_launch_count: returns long long, the binding says int']

    class Narrow(C.Structure):
        _fields_ = _lib.ConvDesc._fields_[:12] + [('slope', C.c_int)] + _lib.ConvDesc._fields_[13:]

    class Swapped(C.Structure):
        _fields_ = [_lib.SmoothDesc._fields_[1], _lib.SmoothDesc._fields_[0]] + _lib.SmoothDesc._fields_[2:]
    bad = binding_mismatches(_lib._SIGS, dict(_lib.STRUCTS, ccb_conv_desc=Narrow, ccb_smooth_desc=Swapped))
    assert bad == ["struct ccb_conv_desc field 12: header ('slope', 'float', ()), ctypes ('slope', 'int', ())",
                   "struct ccb_smooth_desc field 0: header ('kind', 'int', ()), ctypes ('B', 'int', ())"], bad


def test_product_refuses_cpu_tensors_without_simulator():
    import pytest
    import torch
    from cc_b200 import _lib
    if _lib._lib is not None and _lib._is_sim:
        pytest.skip('simulator bound by another test module')
    _lib.use_library(_lib.DEFAULT_PATH)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        _lib.ptr(torch.zeros(4))
    with pytest.raises(RuntimeError, match='ccb_upsample2x_fwd argument 1 .*no CPU fallback'):
        _lib.call('ccb_upsample2x_fwd', None, torch.zeros(4), 1, 1, 1, None)
    with pytest.raises(TypeError, match='ccb_upsample2x_fwd argument 0 must be torch.float32'):
        _lib.call('ccb_upsample2x_fwd', torch.zeros(4, dtype=torch.float64), None, 1, 1, 1, None)
    with pytest.raises(RuntimeError, match=r'ccb_upsample2x_fwd failed \(status -1\): upsample2x_fwd: bad argument'):
        _lib.call('ccb_upsample2x_fwd', None, None, 1, 1, 1, None)       # NULL pointers: refused before any launch
