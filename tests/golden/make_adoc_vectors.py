"""Extracts the example rows of the reference's CEL documentation (docs/modules/policies/pages/conditions.adoc) as test
vectors: every function table there gives, per row, an expression written to hold (evaluate to true) over the section's
"Test data" request fragment.  Needs a cerbos/cerbos source tree (CERBOS_SRC); the output
tests/golden/conditions_adoc.json is committed, this script is how it was made.

    python tests/golden/make_adoc_vectors.py
"""
import json
import os
import re

SRC = os.path.join(os.environ.get("CERBOS_SRC", "."), "docs/modules/policies/pages/conditions.adoc")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "conditions_adoc.json")


def lenient_json(fragment: str):
    """The test-data blocks are JSON object members between '...' lines, with the odd trailing comma."""
    body = "\n".join(l for l in fragment.split("\n") if l.strip() != "...")
    body = re.sub(r",(\s*[}\]])", r"\1", body)
    return json.loads("{" + body.strip().rstrip(",") + "}")


def main():
    lines = open(SRC).read().split("\n")
    section, data, cases = None, {}, []
    i = 0
    while i < len(lines):
        ln = lines[i]
        if ln.startswith("== "):
            section, data = ln[3:].strip(), {}
        elif ln.strip() == ".Test data":
            while lines[i].strip() != "----":
                i += 1
            j = i + 1
            while lines[j].strip() != "----":
                j += 1
            data = lenient_json("\n".join(lines[i + 1:j]))
            i = j
        elif ln.strip() == "|===":
            j = i + 1
            rows, cur = [], None
            while lines[j].strip() != "|===":
                if lines[j].startswith("| "):
                    if cur is not None:
                        rows.append(cur)
                    cur = lines[j]
                elif cur is not None and lines[j].strip():
                    cur += "\n" + lines[j]          # a cell continued on the next line (' +' line breaks)
                j += 1
            if cur is not None:
                rows.append(cur)
            for r in rows[1:]:                      # rows[0] is the header
                cells = [c.strip() for c in r.replace("\\|", "\x00")[1:].split(" | ")]
                if len(cells) < 3:
                    continue
                expr = " ".join(x.strip() for x in cells[-1].replace("\x00", "|").replace(" +\n", "\n").split("\n"))
                cases.append({"section": section, "function": cells[0].strip(), "expr": expr, "request": data, "line": i + 1})
            i = j
        i += 1
    with open(OUT, "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
    print(len(cases), "rows ->", OUT)


if __name__ == "__main__":
    main()
