"""The library's tuning switches (environment variables) are read through one helper, env_knob in common.cuh, and
INTEGRATION §7 documents exactly the switches the sources read."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "galaxysql_b200", "csrc")
HELPER = re.compile(r"template <typename T>\s*static inline bool env_knob\(const char \*name, T \*v\) \{.*?\n\}\n", re.S)


def sources():
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh")):
            with open(os.path.join(CSRC, f)) as fh:
                out[f] = fh.read()
    return out


def knob_names():
    """Names passed to env_knob, and the number of calls (the definition excluded)."""
    names, calls = set(), 0
    for f, src in sources().items():
        if f == "common.cuh":
            src = HELPER.sub("", src)
        calls += len(re.findall(r"\benv_knob\(", src))
        names |= set(re.findall(r"\benv_knob\(\"(GSQL_[A-Z0-9_]+)\"", src))
    return names, calls


def documented_names():
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    section = re.search(r"^## 7\. .*?(?=^## |\Z)", text, re.S | re.M).group(0)
    rows = [line for line in section.splitlines() if line.startswith("| `GSQL_")]
    return {re.match(r"\| `(GSQL_[A-Z0-9_]+)`", row).group(1) for row in rows}, len(rows)


def test_environment_is_read_only_through_env_knob():
    srcs = sources()
    assert len(HELPER.findall(srcs["common.cuh"])) == 1, "env_knob's definition not found in common.cuh"
    for f, src in srcs.items():
        if f == "common.cuh":
            src = HELPER.sub("", src)
        assert "getenv(" not in src, f"{f} reads the environment outside env_knob"


def test_every_switch_read_is_documented_and_every_documented_switch_is_read():
    names, calls = knob_names()
    # every call names its variable literally, so the set above is every switch the library reads
    assert calls == sum(len(re.findall(r"\benv_knob\(\"GSQL_[A-Z0-9_]+\"", s)) for s in sources().values())
    assert calls >= len(names) >= 20
    documented, rows = documented_names()
    assert rows == len(documented), "INTEGRATION §7 lists a switch twice"
    assert names == documented, {"read, not documented": sorted(names - documented), "documented, not read": sorted(documented - names)}
