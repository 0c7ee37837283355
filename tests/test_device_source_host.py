"""The C-ABI of pictures from device memory, without a GPU: the library exports htv_set_video_device_source, and the
ctypes htv_device_frame_t the Python view fills is the C struct, size and offsets as a C compiler lays out the header."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ["width", "height", "data", "stride_x", "stride_y", "stride_c", "serial"]


def test_library_exports_the_setter(built):
    L = built.lib()
    assert hasattr(L, "htv_set_video_device_source")
    assert L.htv_set_video_device_source.argtypes[1] is built._READ_VIDEO_DEVICE


def test_device_frame_layout_matches_the_header(built, tmp_path):
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"hacktv_b200.h\"\nint main(void)\n{\n"
                   "\tprintf(\"%zu\\n\", sizeof(htv_device_frame_t));\n"
                   + "".join(f"\tprintf(\"%zu\\n\", offsetof(htv_device_frame_t, {f}));\n" for f in FIELDS)
                   + "\treturn(0);\n}\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-Wall", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src)])
    got = [int(v) for v in subprocess.check_output([exe], text=True).split()]
    D = built.DeviceFrame
    assert got == [C.sizeof(D)] + [getattr(D, f).offset for f in FIELDS]
    assert [n for n, _ in D._fields_] == FIELDS
