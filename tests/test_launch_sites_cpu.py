"""Every kernel launch in the library goes through launch_kernel / launch_ex (csrc/prof.cuh), which count the launch,
give it its own profile record and name the kernel when the launch fails.  No other source file may launch a kernel
or open a profile scope itself."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'pb_bss_b200', 'csrc')
LAUNCHER = 'prof.cuh'
FORBIDDEN = re.compile(r'<<<|\bLaunchScope\b|\bcudaLaunchKernel\b|\bcudaLaunchKernelEx\b|\bcudaLaunchCooperativeKernel\b')
SOURCES = sorted(f for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh')))


def _code(text):
    """text with its comments and string literals blanked out (line numbers kept)."""
    pattern = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', re.S)
    return pattern.sub(lambda m: '\n' * m.group(0).count('\n'), text)


def test_sources_found():
    assert LAUNCHER in SOURCES
    assert sum(f.startswith('api_') for f in SOURCES) >= 13


def test_launcher_launches():
    code = _code(open(os.path.join(CSRC, LAUNCHER)).read())
    for token in ('<<<', 'LaunchScope', 'cudaLaunchKernelEx'):
        assert token in code


@pytest.mark.parametrize('name', [f for f in SOURCES if f != LAUNCHER])
def test_no_launch_outside_the_launcher(name):
    code = _code(open(os.path.join(CSRC, name)).read())
    found = [(code.count('\n', 0, m.start()) + 1, m.group(0)) for m in FORBIDDEN.finditer(code)]
    assert not found, f'{name}: launch outside {LAUNCHER} at (line, token) {found}'
