"""The option table of csrc/nlt_gconv.cu: every switch's default, how its environment variable is read, what
nlt_set_option stores and what nlt_get_option reads back.  No GPU needed: options are host state, and each
environment spelling runs in a fresh process because an option reads its variable once."""
import ctypes
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'neural-light-transport_b200', 'csrc', 'libnlt_b200.so')


def first_char(ch, val, dflt):
    return lambda e: val if e[:1] == ch else dflt


def atoi(e):
    s = e.lstrip(' \t\n\v\f\r')
    n = len(s) - len(s.lstrip('+-'))
    if n > 1:
        return 0
    digits = s[n:]
    digits = digits[:len(digits) - len(digits.lstrip('0123456789'))]
    return int(s[:n] + digits) if digits else 0


BOOL = lambda v: 1 if v else 0
INT = lambda v: v
NS = lambda v: 2 if v == 2 else 1
TC = lambda v: 0 if v == 0 else (2 if v == 2 else 1)

# name -> (environment variable, value from a set variable, default, stored value of nlt_set_option(v))
ROWS = {
    'tc': ('NLT_DISABLE_TC', first_char('1', 0, 1), 1, TC),
    'tc_wgrad': ('NLT_DISABLE_TC_WGRAD', first_char('1', 0, 1), 1, BOOL),
    'wgrad_rows': (None, None, 1, BOOL),
    'tcs': ('NLT_TCS', lambda e: BOOL(atoi(e)), 1, BOOL),
    'tc_rawhi': ('NLT_TC_RAWHI', first_char('0', 0, 1), 1, BOOL),
    'tc_split_waves': ('NLT_TC_SPLIT_WAVES', first_char('1', 1, 0), 0, BOOL),
    'pwx': ('NLT_PWX', first_char('0', 0, 1), 1, BOOL),
    'pwmma': ('NLT_PWMMA', first_char('0', 0, 1), 1, BOOL),
    'tiny': ('NLT_TINY', first_char('0', 0, 1), 1, BOOL),
    'dconv_cw': ('NLT_DCONV_CW', first_char('0', 0, 1), 1, BOOL),
    'dconv_wide_first': ('NLT_DCONV_WIDE_FIRST', first_char('0', 0, 1), 1, BOOL),
    'pf': ('NLT_PF', first_char('1', 1, 0), 0, BOOL),
    'pf_s1': ('NLT_PF_S1', first_char('1', 1, 0), 0, BOOL),
    'pwd2s_first': ('NLT_PWD2S_FIRST', first_char('1', 1, 0), 0, BOOL),
    'pf_ns': ('NLT_PF_NS', first_char('2', 2, 1), 1, NS),
    'pwx_ns': ('NLT_PWX_NS', first_char('2', 2, 1), 1, NS),
    'wop': ('NLT_WOP', atoi, 1, INT),
    'dconv_wide': ('NLT_DCONV_WIDE', lambda e: BOOL(atoi(e)), 1, BOOL),
    'dconv_wide32': ('NLT_DCONV_WIDE32', atoi, 0, INT),
    'dconv_wide8': ('NLT_DCONV_WIDE8', atoi, 1, INT),
}
# spellings the parsers tell apart: first character 0 / 1 / 2 / other, multi-digit, signs, junk, empty
SPELLINGS = ['0', '1', '2', '10', '21', '-1', '3x', 'on', '']
SET_VALUES = [0, 1, 2, 3, -1, 0]

# Runs in a fresh process: prints {name: [value before any set, value after each nlt_set_option(v)]}.
PROBE = r'''
import ctypes, json, sys
lib = ctypes.CDLL(sys.argv[1])
lib.nlt_set_option.argtypes = [ctypes.c_char_p, ctypes.c_int]
lib.nlt_get_option.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
def get(name):
    v = ctypes.c_int(-12345)
    assert lib.nlt_get_option(name.encode(), ctypes.byref(v)) == 0, name
    return v.value
out = {}
for name in json.loads(sys.argv[2]):
    seq = [get(name)]
    for v in json.loads(sys.argv[3]):
        assert lib.nlt_set_option(name.encode(), v) == 0, name
        seq.append(get(name))
    out[name] = seq
print(json.dumps(out))
'''


def probe(names, set_values=(), **env):
    clean = {k: v for k, v in os.environ.items() if not k.startswith('NLT_')}
    clean.update(env)
    r = subprocess.run([sys.executable, '-c', PROBE, LIB, json.dumps(list(names)), json.dumps(list(set_values))],
                       env=clean, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout)


def test_atoi_restatement():
    assert [atoi(e) for e in ('0', '12', '-3', '+4', ' 5', '3x', 'on', '', '--1')] == [0, 12, -3, 4, 5, 3, 0, 0, 0]


def test_defaults_and_set_get_round_trip():
    got = probe(ROWS, SET_VALUES)
    assert set(got) == set(ROWS)
    for name, (_env, _parse, dflt, store) in ROWS.items():
        assert got[name] == [dflt] + [store(v) for v in SET_VALUES], name
    assert got['tc'][1:4] == [0, 1, 2]          # tc = 2 (every shape the wgmma kernel can run) reads back as 2


@pytest.mark.parametrize('name', [n for n, row in ROWS.items() if row[0] is not None])
def test_environment_spellings(name):
    env, parse, _dflt, _store = ROWS[name]
    for e in SPELLINGS:
        assert probe([name], **{env: e})[name] == [parse(e)], (env, e)


def test_environment_is_read_once_and_set_option_wins():
    # the environment gives the first value; a set replaces it for good
    got = probe(['tc', 'pf'], [1], NLT_DISABLE_TC='1', NLT_PF='1')
    assert got == {'tc': [0, 1], 'pf': [1, 1]}


def test_unknown_and_null_names_are_refused():
    lib = ctypes.CDLL(LIB)
    lib.nlt_set_option.argtypes = [ctypes.c_char_p, ctypes.c_int]
    lib.nlt_get_option.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
    lib.nlt_last_error.restype = ctypes.c_char_p
    v = ctypes.c_int(7)
    assert lib.nlt_set_option(b'no_such_option', 1) == -1
    assert b"unknown option 'no_such_option'" in lib.nlt_last_error()
    assert lib.nlt_get_option(b'no_such_option', ctypes.byref(v)) == -1 and v.value == 7
    assert b"unknown option 'no_such_option'" in lib.nlt_last_error()
    assert lib.nlt_set_option(None, 1) == -1
    assert lib.nlt_get_option(None, ctypes.byref(v)) == -1
    assert lib.nlt_get_option(b'tc', None) == -1


def test_options_context_manager_restores_the_previous_value():
    import nlt_native as nat
    before = {n: nat.get_option(n) for n in ('wop', 'pf_ns', 'tc')}
    with nat.options(wop=2, pf_ns=2, tc=2):
        assert (nat.get_option('wop'), nat.get_option('pf_ns'), nat.get_option('tc')) == (2, 2, 2)
        nat.set_option('wop', 5)
    assert {n: nat.get_option(n) for n in before} == before
    with pytest.raises(ZeroDivisionError):
        with nat.options(tc=0):
            1 / 0
    assert nat.get_option('tc') == before['tc']
    with pytest.raises(nat.NativeError):
        nat.get_option('no_such_option')
