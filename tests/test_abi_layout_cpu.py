"""The ctypes mirror of mpig_config (magicpig_b200._native.MpigConfig) has the header's layout: a small C program compiled
against include/magicpig_b200.h with the host compiler prints the offset and size of every field and the struct's size, and
they must equal the mirror's.  A field the header lacks fails the compile; a swapped, resized or missing field fails the
comparison."""
import ctypes
import os
import shutil
import subprocess

from magicpig_b200 import _native as N


def test_mpig_config_mirror_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    assert cc, "no host C compiler on PATH"
    names = [name for name, _ in N.MpigConfig._fields_]
    lines = "".join(f'    printf("{n} %zu %zu\\n", offsetof(mpig_config, {n}), sizeof(((mpig_config *)0)->{n}));\n' for n in names)
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"magicpig_b200.h\"\n"
                   f"int main(void) {{\n{lines}    printf(\"sizeof %zu 0\\n\", sizeof(mpig_config));\n    return 0;\n}}\n")
    exe = tmp_path / "layout"
    include = os.path.dirname(os.path.abspath(N.HEADER_PATH))
    subprocess.run([cc, "-x", "c", "-std=c99", "-I", include, str(src), "-o", str(exe)], check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    header = {name: (int(off), int(size)) for name, off, size in (line.split() for line in out if line)}
    mirror = {name: (getattr(N.MpigConfig, name).offset, getattr(N.MpigConfig, name).size) for name in names}
    mirror["sizeof"] = (ctypes.sizeof(N.MpigConfig), 0)
    assert mirror == header
