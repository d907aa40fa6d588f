"""Every call of a device entry point in the package goes through _device.call, which checks each argument against
its declaration in include/pbb.h, passes the current stream and raises on a failed call.  No other module may read
the stream for the library or check a return code itself."""
import io
import os
import tokenize

import pytest

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'pb_bss_b200')
BOUNDARY = ('_device.py', '_lib.py')
FORBIDDEN = ('stream_ptr()', '_lib.check(')
SOURCES = sorted(os.path.relpath(os.path.join(d, f), PKG) for d, _, fs in os.walk(PKG) for f in fs if f.endswith('.py'))


def _code(text):
    """text with its comments and string literals blanked out (line numbers kept)."""
    lines = text.splitlines(keepends=True)
    for tok in tokenize.generate_tokens(io.StringIO(text).readline):
        if tok.type in (tokenize.COMMENT, tokenize.STRING):
            (r0, c0), (r1, c1) = tok.start, tok.end
            for r in range(r0, r1 + 1):
                a = c0 if r == r0 else 0
                b = c1 if r == r1 else len(lines[r - 1].rstrip('\n'))
                lines[r - 1] = lines[r - 1][:a] + ' ' * (b - a) + lines[r - 1][b:]
    return ''.join(lines)


def test_sources_found():
    assert all(f in SOURCES for f in BOUNDARY)
    assert len(SOURCES) >= 30


def test_boundary_has_the_protocol():
    code = _code(open(os.path.join(PKG, '_device.py')).read())
    assert 'def call(' in code and '_lib.check(' in code and 'current_stream()' in code


@pytest.mark.parametrize('name', [f for f in SOURCES if f not in BOUNDARY])
def test_no_raw_abi_call_outside_the_boundary(name):
    code = _code(open(os.path.join(PKG, name)).read())
    found = [(i, token) for i, line in enumerate(code.splitlines(), 1) for token in FORBIDDEN if token in line]
    assert not found, f'{name}: raw library call outside _device.call at (line, token) {found}'
