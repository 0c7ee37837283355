"""The C-ABI of sound from device memory, without a GPU: the library exports htv_set_audio_device_source, the header's
htv_device_audio_t and its format codes are what a C compiler lays out and defines, and the ctypes structure the Python
view fills is that struct, size and offsets. The refusal after the first line needs a rendered line, so it is in
tests/test_gpu_zz_device_audio.py."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ["data", "npairs", "format", "stride_pair", "stride_ch"]


def _c_values(tmp_path, body):
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"hacktv_b200.h\"\nint main(void)\n{\n"
                   + body + "\treturn(0);\n}\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src)])
    return [int(v) for v in subprocess.check_output([exe], text=True).split()]


def test_library_exports_the_setter(built):
    L = built.lib()
    assert hasattr(L, "htv_set_audio_device_source")
    assert L.htv_set_audio_device_source.argtypes[1] is built._READ_AUDIO_DEVICE


def test_device_audio_layout_matches_the_header(built, tmp_path):
    got = _c_values(tmp_path, "\tprintf(\"%zu\\n\", sizeof(htv_device_audio_t));\n"
                    + "".join(f"\tprintf(\"%zu\\n\", offsetof(htv_device_audio_t, {f}));\n" for f in FIELDS))
    D = built.DeviceAudio
    assert got == [C.sizeof(D)] + [getattr(D, f).offset for f in FIELDS]
    assert [n for n, _ in D._fields_] == FIELDS
    # the field widths too: a size_t or int64_t declared narrower would still leave the offsets above in place
    widths = _c_values(tmp_path, "".join(f"\tprintf(\"%zu\\n\", sizeof(((htv_device_audio_t *) 0)->{f}));\n"
                                         for f in FIELDS))
    assert widths == [C.sizeof(t) for _, t in D._fields_]


def test_format_codes_match_the_header(built, tmp_path):
    got = _c_values(tmp_path, "\tprintf(\"%d\\n%d\\n\", HTV_PCM_INT16, HTV_PCM_FLOAT32);\n")
    assert got == [built.HTV_PCM_INT16, built.HTV_PCM_FLOAT32]
    assert sorted(built._PCM_FORMATS.values()) == got


def test_setter_refuses_no_encoder(built):
    L = built.lib()
    assert L.htv_set_audio_device_source(None, built._READ_AUDIO_DEVICE(), None) == built.HTV_ERROR
