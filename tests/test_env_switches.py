"""Every environment variable the library or the package reads is one of a short, documented list (DESIGN.md §7).  A path
that replaces another replaces it outright, so a new switch has to be added here and explained there."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / 'novel_view_synthesis_3d_b200'

KEPT = {'XUNET_OP_CACHE_SHADOW', 'XUNET_OP_ATTN_FOLD', 'XUNET_LIB', 'XUNET_CONV_LOG', 'XUNET_NO_PDL',
        'XUNET_NO_SIDE_STREAM', 'XUNET_SM_RESERVE'}


def _read_names():
    names = set()
    for f in sorted((PKG / 'csrc').iterdir()):
        if f.suffix in ('.cu', '.cuh', '.h', '.cpp'):
            names |= set(re.findall(r'getenv\(\s*"(XUNET_[A-Z0-9_]+)"', f.read_text()))
    for f in sorted(PKG.rglob('*.py')):
        names |= set(re.findall(r'os\.environ(?:\.get\(|\.pop\(|\.setdefault\(|\[)\s*[\'"](XUNET_[A-Z0-9_]+)[\'"]',
                                f.read_text()))
    return names


def _design_section_7():
    text = (ROOT / 'DESIGN.md').read_text()
    m = re.search(r'^## 7\..*?(?=^## 8\.)', text, re.M | re.S)
    assert m, 'DESIGN.md has no section 7'
    return m.group(0)


def test_the_library_reads_only_the_kept_environment_variables():
    assert _read_names() == KEPT


def test_every_kept_variable_is_documented_in_design_section_7():
    section = _design_section_7()
    missing = sorted(n for n in KEPT if f'`{n}' not in section)
    assert not missing, missing
