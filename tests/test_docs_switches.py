"""DESIGN.md section 6b lists every run-time switch; each one must exist in the sources it documents (and the header's entry points
must all be bound in _lib.py - that part lives in test_abi.py)."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def _sources() -> str:
    parts = []
    for pat in ("mockingbird_b200/csrc/*.cu", "mockingbird_b200/csrc/*.cpp", "mockingbird_b200/csrc/*.h", "mockingbird_b200/csrc/*.cuh",
                "mockingbird_b200/**/*.py", "*.py", "tools/*.py", "tools/*.sh"):
        for p in ROOT.glob(pat):
            parts.append(p.read_text(errors="ignore"))
    return "\n".join(parts)


def test_every_documented_switch_exists():
    design = (ROOT / "DESIGN.md").read_text()
    sec = design[design.index("## 6b."):design.index("## 7.")]
    names = set()
    for row in sec.splitlines():
        if not row.startswith("| `"):
            continue
        first = row.split("|")[1]
        names.update(re.findall(r"`((?:MB|MOCKINGBIRD)_[A-Z0-9_]+)`", first))
    assert len(names) >= 27, sorted(names)
    src = _sources()
    missing = sorted(n for n in names if n not in src)
    assert not missing, f"documented but not in the sources: {missing}"


def test_every_csrc_switch_is_documented():
    design = (ROOT / "DESIGN.md").read_text()
    used = set()
    for p in (ROOT / "mockingbird_b200" / "csrc").glob("*.cu"):
        used.update(re.findall(r'getenv\("(MB_[A-Z0-9_]+)"\)', p.read_text(errors="ignore")))
    undocumented = sorted(n for n in used if n not in design)
    assert not undocumented, f"getenv switches missing from DESIGN.md: {undocumented}"
