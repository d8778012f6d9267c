"""Compare the SASS of every kernel of two builds of libb2d.so (or two cubins), instruction for instruction.

    python tools/sass_compare.py OLD.so rust-doom_b200/libb2d.so

Runs on a machine without a GPU (cuobjdump + c++filt).  Names are normalised so that a kernel that gained the per-frame
state flag (`kStates`, DESIGN.md §5) is compared, in its `kStates = false` instantiation, with the kernel of the same name
in the old build: the trailing `false` template argument is dropped, and the hash of each anonymous namespace is ignored.
The per-frame level flag (`kLevels`) that follows it is dropped the same way in its `false` instantiations, with the
appended `LevelTables` parameter.  Builds before per-frame states moved into `LevelTables` also took a `StateTables`
parameter ahead of it; that is dropped wherever it stands, so their kernels pair with the later instantiations.
Addresses are dropped; the opcodes and operands are compared.  Exits 1 if any function of OLD is missing from NEW or
differs.
"""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
HEADER = re.compile(r"^(Fatbin |=+$|arch = |code version = |host = |compile_size = |identifier = |code for )")


def functions(path):
    txt = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    txt = subprocess.run(["c++filt"], input=txt, capture_output=True, text=True, check=True).stdout
    txt = re.sub(r"_GLOBAL__N__[0-9a-f_]+_b2d_[a-z]+_cu_[0-9a-f]+", "ANON", txt)
    txt = txt.replace("(anonymous namespace)", "ANON")
    txt = re.sub(r"(b2d_walk_kernel<[a-z]+), false>", r"\1>", txt)
    txt = re.sub(r"(b2d_raster_kernel<[a-z]+, \d+, [a-z]+, [a-z]+), false>", r"\1>", txt)
    txt = re.sub(r"(masked_pass<[a-z]+, \d+, [a-z]+), false>", r"\1>", txt)
    txt = re.sub(r", b2d::LevelTables\)", ")", txt)
    txt = re.sub(r"void (b2d::ANON::b2d_walk_kernel)<false>", r"\1", txt)
    txt = re.sub(r"(b2d_raster_kernel<[a-z]+, \d+, [a-z]+), false>", r"\1>", txt)
    txt = re.sub(r"(masked_pass<[a-z]+, \d+), false>", r"\1>", txt)
    txt = re.sub(r", b2d::StateTables(?=[,)])", "", txt)
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (.*)", line)
        if m:
            cur = m.group(1).strip()
            out[cur] = []
            continue
        line = line.strip()
        if cur is None or not line or HEADER.match(line):
            continue
        ins = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).strip()
        if ins:
            out[cur].append(ins)
    return out


def main():
    if len(sys.argv) != 3:
        raise SystemExit(__doc__)
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    bad = 0
    for name, body in sorted(old.items()):
        if new.get(name) == body:
            print("identical  %6d instructions  %s" % (len(body), name))
        else:
            bad += 1
            print("%s  %s" % ("MISSING   " if name not in new else "DIFFERENT ", name))
    for name in sorted(set(new) - set(old)):
        print("new        %6d instructions  %s" % (len(new[name]), name))
    print("%d of %d functions of %s identical in %s" % (len(old) - bad, len(old), sys.argv[1], sys.argv[2]))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
