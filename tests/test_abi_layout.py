"""The ctypes mirrors in c2m_b200/_lib.py against include/c2m_sm100.h, without the library or a GPU: every struct has the
header's fields in the header's order at the offsets, sizes and total size a C compiler gives them, and every entry
point's argtypes and restype agree with its prototype in count and kind.  A field or argument that drifts out of order
would otherwise make the library read the wrong memory, with nothing to show for it but a wrong number."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from c2m_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'c2m_sm100.h')

STRUCTS = {_lib.DcnShape: 'c2m_dcn_shape', _lib.ConvArgs: 'c2m_conv3x3_args', _lib.DcnTcArgs: 'c2m_dcn_tc_args',
           _lib.DcnTcGradArgs: 'c2m_dcn_tc_grad_args', _lib.PsroiShape: 'c2m_psroi_shape'}

# ctypes type of each scalar C type; every pointer (and the stream handle) is a pointer-sized ctypes type
SCALARS = {'int': ctypes.c_int, 'unsigned': ctypes.c_uint, 'unsigned long long': ctypes.c_ulonglong,
           'long long': ctypes.c_longlong, 'size_t': ctypes.c_size_t, 'float': ctypes.c_float}


def _source():
    return re.sub(r'/\*.*?\*/', '', open(HEADER).read(), flags=re.S)


def _header_structs():
    """{typedef name: [field names in declaration order]}"""
    out = {}
    for body, name in re.findall(r'typedef struct \{(.*?)\}\s*(\w+);', _source(), flags=re.S):
        decls = [d.strip() for d in body.split(';') if d.strip()]
        out[name] = [re.findall(r'\w+', part)[-1] for d in decls for part in d.split(',')]
    return out


def _header_prototypes():
    """{function name: (return type, [parameter types])} with types as written, names dropped."""
    out = {}
    for ret, name, params in re.findall(r'([\w ]+?\**)\s*\b(c2m_\w+)\s*\(([^)]*)\)\s*;', _source()):
        params = [p.strip() for p in params.split(',')]
        types = [] if params == ['void'] else [re.sub(r'\s*\b\w+$', '', p) for p in params]
        out[name] = (ret.strip(), types)
    return out


def _is_pointer(ctype):
    return ctype in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(ctype, ctypes._Pointer)


def _kind(c_type):
    """The ctypes type a C type must map to, or 'pointer'."""
    t = re.sub(r'\bconst\b', '', c_type).strip()
    if '*' in t or t == 'c2m_stream_t':
        return 'pointer'
    return SCALARS[' '.join(t.split())]


def test_every_ctypes_struct_is_mirrored():
    mine = {v for v in vars(_lib).values() if isinstance(v, type) and issubclass(v, ctypes.Structure)}
    assert mine == set(STRUCTS)
    assert set(_header_structs()) == set(STRUCTS.values())


@pytest.mark.skipif(shutil.which('gcc') is None, reason='needs gcc')
def test_struct_layouts_match_the_header(tmp_path):
    fields = _header_structs()
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', 'int main(void) {']
    for cname, names in fields.items():
        lines.append(f'    printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        lines += [f'    printf("{cname} {f} %zu %zu\\n", offsetof({cname}, {f}), sizeof((({cname} *)0)->{f}));'
                  for f in names]
    lines += ['    return 0;', '}']
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines) + '\n')
    subprocess.run(['gcc', '-std=c11', '-Wall', '-Werror', '-o', str(exe), str(src)], check=True)
    c = {}
    for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        cname, what, *vals = ln.split()
        c[cname, what] = tuple(int(v) for v in vals)
    for cls, cname in STRUCTS.items():
        assert [f for f, _ in cls._fields_] == fields[cname], cname
        assert ctypes.sizeof(cls) == c[cname, 'sizeof'][0], cname
        for f, _ in cls._fields_:
            d = getattr(cls, f)
            assert (d.offset, d.size) == c[cname, f], f'{cname}.{f}'


def test_symbol_signatures_match_the_header():
    protos = _header_prototypes()
    assert set(protos) == set(_lib.SYMBOLS)
    for name, (res, args) in _lib.SYMBOLS.items():
        ret, params = protos[name]
        assert len(args) == len(params), name
        for i, (ct, p) in enumerate(zip([res] + args, [ret] + params)):
            want = _kind(p)
            ok = _is_pointer(ct) if want == 'pointer' else ct is want
            assert ok, f'{name}: {"return" if i == 0 else f"argument {i}"} is {ct.__name__}, the header says {p}'
