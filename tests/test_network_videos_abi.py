"""The step-argument struct carries video_grad_scales (one grad scale per video in the packed split step of B
networks' overfits) at the same place in the header and in the ctypes mirror, with the C layout's offsets."""
import ctypes
import re

from conftest import ROOT


def _fields(name):
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "flowmap_b200.h").read_text(), flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\}\s*" + name + ";", text).group(1)
    return [re.findall(r"[A-Za-z_]\w*", part)[-1] for decl in body.split(";") for part in decl.split(",")
            if re.findall(r"[A-Za-z_]\w*", part)]


def test_video_grad_scales_field():
    from flowmap_b200._lib import OverfitStepArgs
    names = [f[0] for f in OverfitStepArgs._fields_]
    assert names == _fields("fm_overfit_step_args")
    i = names.index("video_grad_scales")
    assert names[i - 1:i + 3] == ["metrics_capacity", "video_grad_scales", "B", "gt_fxfy"]
    assert OverfitStepArgs._fields_[i][1] is ctypes.c_int
    # an int between two ints, then the pointer at its 8-byte alignment
    assert OverfitStepArgs.video_grad_scales.offset == OverfitStepArgs.metrics_capacity.offset + 4
    assert OverfitStepArgs.B.offset == OverfitStepArgs.video_grad_scales.offset + 4
    assert OverfitStepArgs.gt_fxfy.offset % 8 == 0
    assert OverfitStepArgs().video_grad_scales == 0  # a zeroed struct keeps the pretraining meaning


def test_struct_offsets_match_the_c_compiler(tmp_path):
    """offsetof / sizeof from the C compiler that builds the library's host code (the one nvcc calls) against
    the ctypes mirror, for the fields around video_grad_scales and for the whole struct."""
    import shutil
    import subprocess
    from flowmap_b200._lib import OverfitStepArgs
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "no C compiler: the library's host code cannot have been built either"
    names = ["metrics_capacity", "video_grad_scales", "B", "gt_fxfy"]
    src = tmp_path / "offsets.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "flowmap_b200.h"\nint main(void) {\n' +
                   "".join(f'  printf("%zu\\n", offsetof(fm_overfit_step_args, {n}));\n' for n in names) +
                   '  printf("%zu\\n", sizeof(fm_overfit_step_args));\n  return 0;\n}\n')
    exe = tmp_path / "offsets"
    subprocess.check_call([cc, "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(OverfitStepArgs, n).offset for n in names] + [ctypes.sizeof(OverfitStepArgs)]
