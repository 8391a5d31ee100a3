"""Every CUDA allocation, stream and event of the library goes through host_stage.cuh: the handles' HandleResources (released in reverse
order of acquisition by the handle's destructor) and HostStage (scratch of the single-frame host entry points).  A direct call anywhere
else is a resource some destroy function has to remember to release.  Host code only, no device."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'sg-slam_b200', 'csrc')

CALLS = re.compile(r'\b(cudaMalloc|cudaMallocHost|cudaFree|cudaFreeHost|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|cudaEventDestroy)\s*\(')
# comments and string / character literals: mentions there are not calls
NOT_CODE = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)


def _calls(path):
    with open(path, encoding='utf-8') as f:
        code = NOT_CODE.sub(lambda m: re.sub(r'[^\n]', ' ', m.group(0)), f.read())
    return [(code.count('\n', 0, m.start()) + 1, m.group(1)) for m in CALLS.finditer(code)]


def test_cuda_resources_are_acquired_only_through_host_stage():
    sources = sorted(f for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh', '.h', '.cpp', '.inc')))
    assert 'host_stage.cuh' in sources and len(sources) > 10
    with open(os.path.join(CSRC, 'host_stage.cuh'), encoding='utf-8') as f:
        owner = f.read()
    assert all(name in owner for name in ('cudaMalloc(', 'cudaMallocHost(', 'cudaFree', 'cudaFreeHost', 'cudaStreamCreateWithFlags(', 'cudaStreamDestroy(',
                                          'cudaEventCreateWithFlags(', 'cudaEventDestroy('))
    stray = [f'{f}:{line}: {name}' for f in sources if f != 'host_stage.cuh' for line, name in _calls(os.path.join(CSRC, f))]
    assert not stray, '\n'.join(stray)


def test_the_scan_sees_calls_and_skips_mentions(tmp_path):
    p = tmp_path / 'x.cu'
    p.write_text('// cudaFree(p) in a comment\nconst char* s = "cudaMalloc(";\n/* cudaEventDestroy(e)\n */ cudaStreamCreateWithFlags (&s, 0);\n'
                 'cudaMallocHost(&h, 4); my_cudaFree(p); cudaMallocAsync(&p, 4, s);\n')
    assert _calls(str(p)) == [(4, 'cudaStreamCreateWithFlags'), (5, 'cudaMallocHost')]
