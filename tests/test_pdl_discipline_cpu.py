"""Programmatic dependent launch (PDL) discipline of every kernel in csrc/, read from the sources.

Every launch goes through xu_launch (common.cuh), which allows the next kernel of the stream to start before the current one
has finished.  That is safe only while each kernel waits for its predecessor (xu_grid_dep_sync: griddepcontrol.wait, then
launch_dependents) before it reads or writes anything global, and before it can leave: a kernel that returns before the wait
lets its successor start while the kernel before it is still running.  So:
  * every __global__ body calls xu_grid_dep_sync() before its first `return`;
  * every kernel calls it first, ahead of any statement but shared-memory and constexpr declarations, except the tensor-core
    kernels listed in PROLOGUE, which set up their shared-memory pipelines (barrier init, fences, tensor-map prefetches of
    their __grid_constant__ maps, fills of shared memory) while the previous kernel drains;
  * such a prologue touches only shared memory, barriers and the tensor maps: no global load, store or atomic, no TMA copy;
  * no kernel is launched with <<<...>>> or a direct cudaLaunchKernel call, only through xu_launch.
"""
import re
from pathlib import Path

import pytest

CSRC = Path(__file__).resolve().parents[1] / 'novel_view_synthesis_3d_b200' / 'csrc'
SOURCES = sorted(p for p in CSRC.iterdir() if p.suffix in ('.cu', '.cuh'))

# kernels whose shared-memory set-up runs ahead of the wait (all six build a TMA / mbarrier pipeline)
PROLOGUE = {'conv_tc_kernel', 'wgrad_tc_kernel', 'pose_dgrad_tc_kernel', 'attn_fwd_tc_kernel', 'attn_bwd_dq_tc_kernel',
            'attn_bwd_dkdv_tc_kernel'}
# what a prologue may call: barrier and fence helpers, index arithmetic, casts
PROLOGUE_CALLS = {'mbar_init', 'fence_async_smem', '__syncthreads', 'reinterpret_cast', 'static_cast', 'min', 'max',
                  'phase_taps', 'attn_cw', 'attn_stages', 'conv_pingpong', 'conv_tbuf_floats', 'sizeof', 'if', 'for', 'while',
                  'asm', 'volatile', 'xu_grid_dep_sync'}
PROLOGUE_ASM = ('fence.mbarrier_init.release.cluster;', 'prefetch.tensormap [%0];')
SHARED_ROOT = 'smem_raw'


def _strip_comments(src):
    src = re.sub(r'/\*.*?\*/', lambda m: '\n' * m.group(0).count('\n'), src, flags=re.S)
    return re.sub(r'//[^\n]*', '', src)


def _match(src, i, open_, close):
    """index just past the bracket closing the one at src[i]"""
    depth = 0
    for j in range(i, len(src)):
        if src[j] == open_:
            depth += 1
        elif src[j] == close:
            depth -= 1
            if depth == 0:
                return j + 1
    raise ValueError('unbalanced')


def kernels():
    """[(file, kernel name, parameter list, body)] of every __global__ function defined in csrc/"""
    out = []
    for path in SOURCES:
        src = _strip_comments(path.read_text())
        for m in re.finditer(r'__global__\b', src):
            # the name is the identifier right before the parameter list's '(' (after any __launch_bounds__(..) etc.)
            i = m.end()
            name = None
            while True:
                nm = re.compile(r'\s*([A-Za-z_]\w*)\s*(\()').match(src, i)
                if nm is None:
                    nm2 = re.compile(r'\s*[^;{(]*?([A-Za-z_]\w*)\s*\(').search(src, i)
                    i = nm2.start(1)
                    continue
                j = _match(src, nm.start(2), '(', ')')
                rest = re.compile(r'\s*(\{|;)').match(src, j)
                if nm.group(1) in ('__launch_bounds__', '__cluster_dims__') or rest is None:
                    i = j
                    continue
                name, params = nm.group(1), src[nm.start(2) + 1:j - 1]
                if rest.group(1) == ';':
                    name = None       # a declaration; the definition is found on its own
                else:
                    body = src[rest.start(1) + 1:_match(src, rest.start(1), '{', '}') - 1]
                break
            if name is not None:
                out.append((path.name, name, params, body))
    return out


KERNELS = kernels()
IDS = [f'{f}:{n}' for f, n, _, _ in KERNELS]
SYNC = re.compile(r'\bxu_grid_dep_sync\s*\(\s*\)\s*;')


def _statements(body):
    """top-level statements of a body, up to and including the first xu_grid_dep_sync(); nested blocks kept whole"""
    out, i, start = [], 0, 0
    while i < len(body):
        c = body[i]
        if c == '{':
            i = _match(body, i, '{', '}')
            if re.match(r'\s*(if|for|while|else)\b', body[start:]) or body[start:i].strip().startswith('{'):
                nxt = re.compile(r'\s*else\b').match(body, i)
                if nxt:
                    i = nxt.end()
                    continue
                out.append(body[start:i].strip())
                start = i
            continue
        if c == '(':
            i = _match(body, i, '(', ')')
            continue
        if c == ';':
            out.append(body[start:i + 1].strip())
            start = i + 1
        i += 1
    return [s for s in out if s]


def test_the_kernel_list_is_complete():
    """the parser sees every __global__ of the sources (a kernel it skipped would go unchecked)"""
    n = sum(len(re.findall(r'__global__\b', _strip_comments(p.read_text()))) for p in SOURCES)
    assert len(KERNELS) == n, (len(KERNELS), n)
    assert len(KERNELS) >= 50
    assert PROLOGUE <= {k for _, k, _, _ in KERNELS}


@pytest.mark.parametrize('kernel', KERNELS, ids=IDS)
def test_kernel_waits_before_its_first_return(kernel):
    f, name, _, body = kernel
    s = SYNC.search(body)
    assert s is not None, f'{f}:{name} never calls xu_grid_dep_sync()'
    r = re.search(r'\breturn\b', body)
    assert r is None or r.start() > s.start(), f'{f}:{name} can return before xu_grid_dep_sync()'


@pytest.mark.parametrize('kernel', [k for k in KERNELS if k[1] not in PROLOGUE], ids=[i for i, k in zip(IDS, KERNELS) if k[1] not in PROLOGUE])
def test_kernel_waits_first(kernel):
    f, name, _, body = kernel
    for st in _statements(body):
        if SYNC.fullmatch(st):
            return
        # only declarations without effects may come first: dynamic / static shared memory, compile-time constants
        assert re.match(r'(extern\s+)?__shared__\b|(static\s+)?constexpr\b', st), f'{f}:{name} runs `{st[:80]}` before xu_grid_dep_sync()'
    pytest.fail(f'{f}:{name}: no top-level xu_grid_dep_sync()')


def _prologue(body):
    s = SYNC.search(body)
    return body[:s.start()]


@pytest.mark.parametrize('name', sorted(PROLOGUE))
def test_prologue_touches_only_shared_memory_barriers_and_tensor_maps(name):
    (f, _, params, body), = [k for k in KERNELS if k[1] == name]
    raw = _prologue(body)
    pro = re.sub(r'"[^"]*"', '""', raw)       # the asm strings are checked on their own below
    # every pointer the prologue declares derives from the dynamic shared memory
    shared = {SHARED_ROOT}
    for m in re.finditer(r'([A-Za-z_]\w*)\s*\*\s*([A-Za-z_]\w*)\s*=\s*([^;]*);', pro):
        refs = set(re.findall(r'[A-Za-z_]\w*', m.group(3)))
        assert refs & shared, f'{f}:{name}: prologue pointer {m.group(2)} = {m.group(3)} is not shared memory'
        shared.add(m.group(2))
    local_arrays = set(re.findall(r'\b(?:int|float|uint32_t)\s+([A-Za-z_]\w*)\s*\[', pro))
    local_arrays |= set(re.findall(r',\s*([A-Za-z_]\w*)\s*\[\s*\d+\s*\]', pro))
    # indexing or dereferencing: shared pointers and local arrays only (never a kernel parameter's pointer)
    for m in re.finditer(r'([A-Za-z_][\w.]*)\s*\[', pro):
        base = m.group(1)
        assert base in shared or base in local_arrays, f'{f}:{name}: prologue indexes {base}[...]'
    # calls: barrier / fence helpers and index arithmetic only
    for m in re.finditer(r'([A-Za-z_]\w*)\s*(?:<[^<>;]*>)?\s*\(', pro):
        assert m.group(1) in PROLOGUE_CALLS or m.group(1) in ('uint8_t', 'uint32_t', 'uint64_t', 'uintptr_t', 'float', 'int', 'size_t'), \
            f'{f}:{name}: prologue calls {m.group(1)}()'
    for m in re.finditer(r'asm\s+volatile\s*\(\s*"([^"]*)"', raw):
        assert m.group(1) in PROLOGUE_ASM, f'{f}:{name}: prologue runs `{m.group(1)}`'
    # tensor-map prefetches name __grid_constant__ parameters
    grid_const = set(re.findall(r'__grid_constant__\s+CUtensorMap\s+([A-Za-z_]\w*)', params))
    for m in re.finditer(r'prefetch\.tensormap[^:]*::"l"\(&([A-Za-z_]\w*)\)', raw):
        assert m.group(1) in grid_const, f'{f}:{name}: prefetches {m.group(1)}, not a __grid_constant__ tensor map'
    # nothing global: no TMA copy, load, store, atomic or reduction
    for bad in (r'\btma_\w*\s*\(', r'\bld\.global', r'\bst\.global', r'\batomic', r'\bred\.', r'\bcp\.async', r'__ldg', r'xu_det_add'):
        assert not re.search(bad, raw), f'{f}:{name}: prologue uses {bad}'


def test_every_launch_goes_through_xu_launch():
    for path in SOURCES:
        src = _strip_comments(path.read_text())
        assert '<<<' not in src, f'{path.name} launches a kernel with <<<...>>>'
        for m in re.finditer(r'\b(cudaLaunchKernel(?:Ex)?|cudaLaunchCooperativeKernel|cuLaunchKernel(?:Ex)?)\s*\(', src):
            # the one launch site: xu_launch in common.cuh
            assert path.name == 'common.cuh', f'{path.name} calls {m.group(1)} directly'
    common = _strip_comments((CSRC / 'common.cuh').read_text())
    assert len(re.findall(r'\bcudaLaunchKernelEx\s*\(', common)) == 1
