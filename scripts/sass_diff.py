"""Compare the SASS of every conv_tc_kernel instance between two object files (addresses stripped): used to show that
adding opt-in kernel variants left the GPU-validated default instances bit-identical, or that moving shared helpers
into common.cuh left a file's kernels unchanged (any object file; kernels in an anonymous namespace match by name).

    python scripts/sass_diff.py old_conv_tc.o keras-ocr_b200/csrc/conv_tc.o [suffix-to-append-to-old-template-args]

e.g. after a new trailing template parameter `bool BOX16 = false` pass `ELb0` so that old `<64,64,3,true>` is compared
with new `<64,64,3,true,false>`.  A kernel that became a template, or gained parameters, is matched by an argument
OLD=NEW that renames it (substrings of the mangled names), e.g.

    python scripts/sass_diff.py old_ctc_beam.o new_ctc_beam.o \
        ctc_beam_lm_kernelEPKfiiiPKyS1_iiffPiPfS5_=ctc_beam_lm_kernelILb0EEEvPKfiiiPKyS2_iiffPiPfS6_NS_4TrieE
"""
import collections
import re
import subprocess
import sys


def functions(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    table, name = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            full = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", m.group(1))   # anonymous namespace: per-build hash
            full = re.sub(r"(_GLOBAL__N__\d+_\w+?_cu)_[0-9a-f]{8}", r"\1_", full)  # and the hash of the file's contents
            # conv_tc_kernel instances are named by their template arguments; other templates keep their full name
            name = full[full.index("kernelI"):] if "conv_tc_kernelI" in full else full
            table[name] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and name:
            table[name].append(re.sub(r"\s+", " ", m.group(1)))
    return table


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    extra = sys.argv[3:]
    renames = [tuple(a.split("=", 1)) for a in extra if "=" in a]
    suffix = next((a for a in extra if "=" not in a), "")
    same = 0
    for name, body in old.items():
        other = name.replace("EEEv14CUtensorMap", suffix + "EEEv14CUtensorMap") if suffix else name
        for a, b in renames:
            other = other.replace(a, b)
        if body == new.get(other):
            same += 1
        else:
            print("DIFFERENT" if other in new else "MISSING  ", name[:60])
    print(f"{same} of {len(old)} instances identical; {len(new) - len(old)} instances only in the second file")


if __name__ == "__main__":
    main()
