#!/usr/bin/env python3
"""Extract golden vectors from the reference's playthrough traces.

Reads open_spiel/integration_tests/playthroughs/<game>.txt of the OpenSpiel checkout
__graft_entry__.REFERENCE (the
line-for-line golden traces checked by the reference's
integration_tests/playthrough_test.py:73-98; format defined by
python/algorithms/generate_playthrough.py:211-521) and writes one compact JSON
fixture per trace under tests/golden/playthroughs/.

Only this script reads the reference; the tests read the committed JSON.

JSON layout:
  {"game": "<game string>", "header": {"NumDistinctActions": 7, ...},
   "actions": [a0, a1, ...],                       # the applied action ids
   "states": [ {"index": k, "to_string": "...", "detailed": bool,
                "is_terminal": bool, "current_player": int,
                "legal_actions": [...], "returns": [...], "rewards": [...],
                "chance_outcomes": [[a, p], ...],
                "strings": {"InformationStateString(0)": "...", ...},
                "tensors": {"ObservationTensor(0)": [flat floats], ...}} ]}
Tensors are flattened in the order the trace prints them: for structured
(multi-field) observers the fields are concatenated in print order, which is the
ContiguousAllocator order (observer.h:174-186).
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from __graft_entry__ import REFERENCE  # noqa: E402

REF = os.path.join(REFERENCE, "open_spiel", "integration_tests", "playthroughs")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "playthroughs")

TRACES = [
    "tic_tac_toe", "connect_four", "breakthrough", "hex(board_size=5)", "go",
    "kuhn_poker_2p", "leduc_poker_1540482260", "leduc_poker_3977671846",
    "leduc_poker_773740114", "kuhn_poker_3p", "leduc_poker_3p",
    "mnk", "othello", "y(board_size=9)", "havannah(board_size=4)", "havannah(board_size=4,swap=True)",
]

CIRCLES = {"◯": 0.0, "◉": 1.0}


def _is_circle_row(s):
    t = s.replace(" ", "")
    return bool(t) and all(ch in CIRCLES for ch in t)


def _parse_circle_block(first_inline, following):
    """Return flat floats from a printed 1/2/3-D 0/1 tensor.

    first_inline: text after 'name:' on the header line ('' for 3-D tensors).
    following: continuation lines (already stripped of the newline).
    """
    rows = []
    if first_inline.strip():
        rows.append(first_inline.strip())
    rows.extend(r.strip() for r in following if r.strip())
    # 3-D tensors print planes side by side separated by two spaces; several
    # "big rows" of planes may be stacked, separated by a blank line (kept out
    # of `following` by the caller, which passes groups).
    planes = None
    for r in rows:
        parts = r.split("  ")
        if planes is None:
            planes = [[] for _ in parts]
        for p, part in zip(planes, parts):
            p.append([CIRCLES[ch] for ch in part])
    flat = []
    for p in planes or []:
        for row in p:
            flat.extend(row)
    return flat


def parse(path):
    with open(path, encoding="utf-8") as f:
        lines = f.read().split("\n")
    out = {"game": None, "header": {}, "actions": [], "states": []}
    i = 0
    assert lines[0].startswith("game: ")
    out["game"] = lines[0][len("game: "):]
    i = 1
    # header
    while i < len(lines) and not lines[i].startswith("# State "):
        m = re.match(r"^(\w+)\(\) = (.*)$", lines[i])
        if m:
            out["header"][m.group(1)] = m.group(2)
        i += 1
    cur = None
    while i < len(lines):
        ln = lines[i]
        if ln.startswith("# State "):
            cur = {"index": int(ln[len("# State "):]), "to_string_lines": [],
                   "detailed": False, "strings": {}, "tensors": {}}
            out["states"].append(cur)
            i += 1
            while i < len(lines) and lines[i].startswith("#") and not \
                    lines[i].startswith("# Apply action") and not lines[i].startswith("# State "):
                cur["to_string_lines"].append(lines[i][2:] if lines[i].startswith("# ") else lines[i][1:])
                i += 1
            continue
        if ln.startswith("action: "):
            out["actions"].append(int(ln[len("action: "):]))
            i += 1
            continue
        if ln.startswith("# Apply action") or ln == "":
            i += 1
            continue
        m = re.match(r"^(IsTerminal|CurrentPlayer|IsChanceNode)\(\) = (.*)$", ln)
        if m:
            cur["detailed"] = True
            key, val = m.group(1), m.group(2)
            if key == "IsTerminal":
                cur["is_terminal"] = (val == "True")
            elif key == "IsChanceNode":
                cur["is_chance"] = (val == "True")
            else:
                cur["current_player"] = int(val)
            i += 1
            continue
        m = re.match(r"^(LegalActions|Returns|Rewards|History)\(\) = \[(.*)\]$", ln)
        if m:
            key = {"LegalActions": "legal_actions", "Returns": "returns",
                   "Rewards": "rewards", "History": "history"}[m.group(1)]
            body = m.group(2).strip()
            vals = [float(x) if key in ("returns", "rewards") else int(x)
                    for x in body.split(",")] if body else []
            if key in ("returns", "rewards"):
                # keep the sign of negative zero ("-0") visible
                cur[key + "_text"] = [x.strip() for x in body.split(",")] if body else []
            cur[key] = vals
            i += 1
            continue
        m = re.match(r"^ChanceOutcomes\(\) = \[(.*)\]$", ln)
        if m:
            cur["chance_outcomes"] = [[int(a), float(p)] for a, p in
                                      re.findall(r"\((\d+),([0-9.eE+-]+)\)", m.group(1))]
            i += 1
            continue
        m = re.match(r"^((?:Observation|InformationState)Tensor\(\d+\))(\.\w+)?(: ?| = )(.*)$", ln)
        if m:
            name = m.group(1)
            sep, rest = m.group(3), m.group(4)
            vals = None
            if sep.strip() == "=":
                vals = [float(x) for x in rest.strip()[1:-1].split(",") if x.strip()]
                i += 1
            else:
                i += 1
                vals = []
                first = rest
                while True:
                    group = []
                    while i < len(lines) and _is_circle_row(lines[i]):
                        group.append(lines[i])
                        i += 1
                    vals.extend(_parse_circle_block(first, group))
                    first = ""
                    # stacked big-rows of a 3-D tensor: blank line then more circle rows
                    if i + 1 < len(lines) and lines[i] == "" and _is_circle_row(lines[i + 1]):
                        i += 1
                        continue
                    break
            cur["tensors"].setdefault(name, []).extend(vals)
            continue
        m = re.match(r"^(\w+String\(\d*\)) = (.*)$", ln)
        if m:
            try:
                cur["strings"][m.group(1)] = json.loads(m.group(2))
            except Exception:
                cur["strings"][m.group(1)] = m.group(2)
            i += 1
            continue
        i += 1
    for s in out["states"]:
        s["to_string"] = "\n".join(s.pop("to_string_lines"))
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    for name in TRACES:
        src = os.path.join(REF, name + ".txt")
        data = parse(src)
        data["source"] = "open_spiel/integration_tests/playthroughs/%s.txt" % name
        dst = os.path.join(OUT, name + ".json")
        with open(dst, "w", encoding="utf-8") as f:
            json.dump(data, f, separators=(",", ":"), ensure_ascii=False)
        nd = sum(1 for s in data["states"] if s["detailed"])
        print("%-28s game=%-45s states=%d detailed=%d actions=%d" % (
            name, data["game"], len(data["states"]), nd, len(data["actions"])))


if __name__ == "__main__":
    sys.exit(main())
