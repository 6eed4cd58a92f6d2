"""Documentation that must not drift from the code."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _read(*parts):
    with open(os.path.join(ROOT, *parts), encoding="utf-8") as f:
        return f.read()


def test_every_environment_switch_is_documented_in_the_readme():
    """Every CT2B200_* variable the product reads with getenv / os.environ appears in README.md's table."""
    used = set()
    for base, _, files in os.walk(os.path.join(ROOT, "ctranslate2_b200")):
        if "_build" in base or "__pycache__" in base:
            continue
        for name in files:
            if name.endswith((".cu", ".cuh", ".cc", ".h", ".py")):
                text = _read(base, name)
                used |= set(re.findall(r'(?:getenv|env_int|env_mb|environ\.get)\(\s*"(CT2B200_[A-Z0-9_]+)"', text))
    used |= set(re.findall(r'environ\.get\(\s*"(CT2B200_[A-Z0-9_]+)"', _read("bench.py")))
    assert used, "no environment switches found: the scan is broken"
    readme = _read("README.md")
    missing = sorted(v for v in used if v not in readme)
    assert not missing, "undocumented environment switches: %s" % missing


def test_design_and_integration_cite_existing_files():
    """Paths of this repository named in DESIGN.md / INTEGRATION.md / README.md exist."""
    pat = re.compile(r"`((?:ctranslate2_b200|oracle|tests|tools|include)/[A-Za-z0-9_./-]+\.(?:cu|cuh|cc|h|py|md|sh|json|csv))`")
    for doc in ("DESIGN.md", "INTEGRATION.md", "README.md"):
        for path in pat.findall(_read(doc)):
            assert os.path.exists(os.path.join(ROOT, path)), "%s cites a missing file: %s" % (doc, path)
