"""The picture-row table of the converted picture store (htv_tables.c build_pic_rows), without a GPU: for every mode, with
and without `interlaced`, it is the inverse of the line -> source row map the raster descriptors use (line_numbers,
ref video.c:2812-2895), and each row carries the picture area of the line that shows it."""
import pytest

def _modes(H):
    return sorted(H.modes())


def _vy(conf, line):
    # the source row of `line` (1-based): line_numbers / htv_line_vy, restated
    if conf.lines == 625:
        vy = (line - 23) * 2 if line < 313 else (line - 336) * 2 + 1
    else:
        vy = (line - 23) * 2 if line < 265 else (line - 286) * 2 + 1
    if vy >= 0 and conf.interlaced:
        vy += 1
    return vy if 0 <= vy < conf.active_lines else -1


@pytest.mark.parametrize("interlaced", [1, 0])
def test_picture_rows_invert_the_line_map_for_every_mode(built, interlaced):
    H = built
    checked = 0
    for mode in _modes(H):
        conf = H.mode_config(mode)
        conf.interlaced = interlaced
        rate = 16000000 if conf.lines == 625 else 13500000
        try:
            t = H.Tables(conf, rate)
        except RuntimeError:
            continue                                             # not on the accelerated path
        codes, geo = t.get("codes"), t.get("geometry")
        rows, line_row = t.get("pic_rows").reshape(-1, 4), t.get("line_row")
        t.close()
        W, half, aleft, awidth = (int(v) for v in geo[:4])
        al_n = conf.active_lines
        assert len(line_row) == conf.lines + 1 and line_row[0] == -1 and len(rows) >= al_n, mode
        shown = set()
        for line in range(1, conf.lines + 1):
            left, right = codes[line] & (1 << 7), codes[line] & (1 << 8)
            vy, r = _vy(conf, line), int(line_row[line])
            if not left and not right:
                assert r == -1, (mode, line)
                continue
            # a line with a picture area shows its source row, or (none) a black row of its own behind the picture rows
            assert r == vy if vy >= 0 else r >= al_n, (mode, line, vy, r)
            assert r not in shown, (mode, line)
            shown.add(r)
            al = aleft if left else half
            ar = aleft + awidth if right else half
            assert list(rows[r][:3]) == [line, al, ar], (mode, line, list(rows[r]))
        # every other row is drawn by no line
        for r in range(len(rows)):
            if r not in shown:
                assert list(rows[r]) == [0, 0, 0, 0], (mode, r)
        assert len(rows) == al_n + sum(1 for r in shown if r >= al_n), mode
        checked += 1
    assert checked >= 20
