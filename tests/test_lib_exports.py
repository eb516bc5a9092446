"""CPU-side checks of the boundary: the shared library is present, loads, and exports every
symbol include/surreal_b200.h declares.  No compute calls (no GPU here)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    txt = open(os.path.join(ROOT, 'include', 'surreal_b200.h')).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    return sorted(set(re.findall(r'\b(sb200_[a-z0-9_]+)\s*\(', txt)))


def test_library_builds_loads_and_exports_header_symbols():
    from surreal_b200 import build, _lib
    build.build()
    L = _lib.lib()
    syms = _header_symbols()
    assert len(syms) >= 5
    for s in syms:
        assert hasattr(L, s), 'header declares %s but the library does not export it' % s
    declared = set(_lib.exported_symbols())
    assert set(syms) == declared, 'ctypes signatures out of sync with the header: %s' % (set(syms) ^ declared)
    assert L.sb200_version() >= 100
    assert L.sb200_status_string(-1) == b'invalid argument'


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from surreal_b200 import _lib
    monkeypatch.setattr(_lib, '_lib', None)
    monkeypatch.setattr(_lib, 'LIB_PATH', str(tmp_path / 'nope.so'))
    with pytest.raises(_lib.SB200Error):
        _lib.lib()


def _header_prototypes():
    """{symbol: [C parameter type strings]} parsed from the header (comments stripped)."""
    txt = open(os.path.join(ROOT, 'include', 'surreal_b200.h')).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    protos = {}
    for m in re.finditer(r'\b(sb200_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;', txt, flags=re.S):
        params = [p.strip() for p in m.group(2).replace('\n', ' ').split(',')]
        if params == ['void'] or params == ['']:
            params = []
        protos[m.group(1)] = params
    return protos


def test_ctypes_signatures_match_header_prototypes():
    """Arity and pointer-vs-scalar class of every ctypes signature against the C prototype: a miscounted argument list
    would otherwise only show up as garbage on the GPU box."""
    import ctypes as C
    from surreal_b200 import _lib
    L = _lib.lib()
    protos = _header_prototypes()
    assert len(protos) >= 40
    ptr_like = (C.c_void_p, C.c_char_p)
    for name, params in protos.items():
        fn = getattr(L, name)
        argtypes = fn.argtypes or []
        assert len(argtypes) == len(params), '%s: header has %d parameters, ctypes %d' % (name, len(params), len(argtypes))
        for i, (ct, cp) in enumerate(zip(argtypes, params)):
            is_ptr_c = '*' in cp
            is_ptr_py = ct in ptr_like or hasattr(ct, 'contents') or (hasattr(ct, '_type_') and not isinstance(ct._type_, str))
            assert is_ptr_c == bool(is_ptr_py), '%s arg %d: header "%s" vs ctypes %s' % (name, i, cp, ct)
            if not is_ptr_c:
                want = ('double', 'float') if ct in (C.c_double, C.c_float) else ('int', 'int64_t', 'uint64_t', 'size_t')
                assert cp.split()[0] in want or cp.split()[-2] in want, '%s arg %d: header "%s" vs ctypes %s' % (name, i, cp, ct)


# header struct -> ctypes Structure of surreal_b200._lib (None: no binding, the struct is only ever device memory)
STRUCTS = {'sb200_mlp': 'Mlp', 'sb200_zfilter': 'ZFilter', 'sb200_rows': 'Rows', 'sb200_par': 'Par',
           'sb200_epochs': 'Epochs', 'sb200_windows': 'Windows', 'sb200_window_rows': 'WindowRows',
           'sb200_ppo_act': 'PPOAct', 'sb200_ddpg_act': 'DDPGAct', 'sb200_dqn_agent_act': 'DQNAgentAct',
           'sb200_ppo_rollout': 'PPORollout', 'sb200_ssar': 'Ssar', 'sb200_env': 'Env', 'sb200_param_noise_state': None}


def _header_structs():
    """{struct name: [(field, C type)]} of every `typedef struct { ... } sb200_*;` in the header (comments stripped); a
    pointer declarator puts '*' in the type, an array declarator keeps only its element type."""
    txt = open(os.path.join(ROOT, 'include', 'surreal_b200.h')).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    structs = {}
    for m in re.finditer(r'typedef\s+struct\s*\{(.*?)\}\s*(sb200_\w+)\s*;', txt, flags=re.S):
        fields = []
        for decl in filter(None, (d.strip() for d in m.group(1).split(';'))):
            base, first = re.match(r'((?:const\s+)?\w+)\s*(.*)$', decl, flags=re.S).groups()
            for d in first.split(','):
                stars, name = re.match(r'\s*(\**)\s*(\w+)\s*(?:\[[^\]]*\])?\s*$', d).groups()
                fields.append((name, base.replace('const', '').strip() + stars))
        structs[m.group(2)] = fields
    return structs


def test_ctypes_structures_match_header_structs():
    """Field names, order and class of every ctypes Structure against the header's struct: pointer fields (any pointer
    type), scalar fields (the exact C type) and nested structs (the bound ctypes type).  A swapped or missing field would
    otherwise only show up as garbage on the GPU box."""
    import ctypes as C
    from surreal_b200 import _lib
    scalars = {'int': C.c_int, 'int64_t': C.c_int64, 'uint64_t': C.c_uint64, 'uint32_t': C.c_uint32, 'float': C.c_float,
               'double': C.c_double}
    structs = _header_structs()
    assert set(structs) == set(STRUCTS), 'header structs without a binding decision: %s' % (set(structs) ^ set(STRUCTS))
    for cname, pyname in STRUCTS.items():
        if pyname is None:
            continue
        py = getattr(_lib, pyname)
        header = structs[cname]
        assert [f[0] for f in py._fields_] == [f[0] for f in header], '%s vs %s: field names / order differ' % (cname, pyname)
        for (field, ct), (_, ctype) in zip(py._fields_, header):
            while issubclass(ct, C.Array):
                ct = ct._type_
            what = '%s.%s: header "%s" vs ctypes %s' % (cname, field, ctype, ct)
            if ctype.endswith('*'):
                assert ct in (C.c_void_p, C.c_char_p) or issubclass(ct, C._Pointer), what
            elif ctype in STRUCTS:
                assert ct is getattr(_lib, STRUCTS[ctype]), what
            else:
                assert ct is scalars[ctype], what
