"""Every `file.py:NN[-MM]` citation of a reference file in the product, the oracle, the tests and the docs points INSIDE that file
Range check only - what the lines say is the reviewer's job.  The line counts of the reference's .py / .yaml / .txt / .toml
files (per base name) are stored in tests/golden/reference_line_counts.json."""
import glob
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAT = re.compile(r"([A-Za-z0-9_]+\.(?:py|yaml|txt|toml)):(\d+)(?:[-–](\d+))?((?:,\s*\d+(?:[-–]\d+)?)*)")


def test_reference_citations_are_inside_the_cited_files():
    with open(os.path.join(ROOT, "tests", "golden", "reference_line_counts.json")) as f:
        lengths = json.load(f)
    files = [p for pat in ("easyanimate_b200/**/*.py", "easyanimate_b200/csrc/*.cu*", "easyanimate_b200/csrc/*.h", "include/*.h",
                           "oracle/**/*.py", "tests/**/*.py", "tools/*.py", "*.md", "bench.py", "__graft_entry__.py")
             for p in glob.glob(os.path.join(ROOT, pat), recursive=True)
             if os.path.basename(p) not in ("PAPERS.md", "SNIPPETS.md")]
    checked, bad = 0, []
    for path in files:
        with open(path, errors="replace") as f:
            text = f.read()
        for m in PAT.finditer(text):
            name = m.group(1)
            if name not in lengths:
                continue  # a file of this repository, not of the reference
            last = max(int(x) for x in re.findall(r"\d+", m.group(0)[len(name) + 1:]))
            checked += 1
            if all(last > n for n in lengths[name]):
                bad.append(f"{os.path.relpath(path, ROOT)}: {m.group(0)} (longest {name}: {max(lengths[name])} lines)")
    assert checked > 200 and not bad, bad
