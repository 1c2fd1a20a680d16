"""cv::resize on the device held to the C port (oracle/port/port_geometry.c) bit for bit -- NaN as NaN, every other float by its bits --
over the table of tests/resize_cases.py.  tests/test_resize_port.py holds the port to the reference over the same table, so nothing
here needs the reference and nothing skips.

About twenty kernels share the work (opencv_b200/csrc/resize*.cu) and resize_impl chooses among them by interpolation, type, size,
alignment and two switches.  Every case runs through the default dispatch; NEAREST also through B200CV_RESIZE_NN_PATH=v1 and =walk,
8-bit LANCZOS4 through B200CV_RESIZE_LANCZOS_PATH=v1.  resize_cases.predict() restates the dispatch; test_predicted_kernel_runs
checks it, template arguments and the tiled kernels' row blocks included, against the kernels torch.profiler sees.

A failure names the path, the kernel, the case, the first differing element and where it sits: its tile column and row block, its
place in the 4-element item, and whether it lies in the reference's vector body or its scalar tail.
"""
import json
import re

import numpy as np
import pytest

import opencv_b200 as C
import resize_cases as rc

pytestmark = pytest.mark.gpu

U8_FILL, F32_FILL = 0xA5, -777.25
ENV = {"nn": "B200CV_RESIZE_NN_PATH", "lz": "B200CV_RESIZE_LANCZOS_PATH"}


def paths_of(case):
    if case.interp == rc.NEAREST:
        return (None, ("nn", "v1"), ("nn", "walk"))
    if case.interp == rc.LANCZOS4 and case.dtype == "u8":
        return (None, ("lz", "v1"))
    return (None,)


def set_path(monkeypatch, path):
    for v in ENV.values():
        monkeypatch.delenv(v, raising=False)
    if path is not None:
        monkeypatch.setenv(ENV[path[0]], path[1])


def device_resize(cvb, case, src, dst=None):
    if case.fxfy is not None:
        return cvb.resize(src, None, case.fxfy[0], case.fxfy[1], case.interp, dst=dst)
    return cvb.resize(src, case.dsize, interpolation=case.interp, dst=dst)


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def to_host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def assert_same(got, want, case, path, what="", **align):
    """got == want for one frame, (h, w) or (h, w, cn)"""
    got = np.asarray(got).reshape(want.shape)
    if rc.same(got, want):
        return
    bad = np.argwhere(rc.differs(got, want))
    y, x = int(bad[0][0]), int(bad[0][1])
    c = int(bad[0][2]) if got.ndim == 3 else 0
    pred = rc.predict(case, path, **align)
    tw, th = rc.tile_of(pred)
    e = x * case.cn + c
    body = rc.body_limit(case, pred)
    where = "tile column %d (%d columns), row block %d (%d rows), element %d of its 4-element item, %s" % (
        x // tw, tw, y // th, th, e % 4, "vector body" if body is None or e < body else "scalar tail (from element %d)" % body)
    g, w = rc.canonical(got)[tuple(bad[0])], rc.canonical(want)[tuple(bad[0])]
    raise AssertionError("path %s, kernel %s%s, case %s%s: %d of %d elements differ, first at y = %d, x = %d, c = %d: got %r want %r; %s" % (
        "default" if path is None else "%s=%s" % (ENV[path[0]], path[1]), pred.kernel, pred.args, case.id, what, len(bad), got.size,
        y, x, c, g, w, where))


# ---------------------------------------------------------------------------------------------------------------- the whole table
@pytest.mark.parametrize("case", rc.CASES, ids=lambda c: c.id)
def test_kernels_vs_port(cvb, port, monkeypatch, case):
    import torch
    frames = rc.frames_of(case)
    want = [rc.run(port, case, f) for f in frames]
    dw, dh = case.dsize
    tdt = torch.uint8 if case.dtype == "u8" else torch.float32
    if case.frames == 1:
        src = dev(frames[0])
    else:
        # a batch whose frame stride is larger than a frame: (N, h + 2, w, cn)[:, :h], and (N, dh + 3, dw, cn)[:, :dh] for the destination
        h, w = case.src
        src = torch.full((case.frames, h + 2, w, case.cn), 99, dtype=tdt, device="cuda")[:, :h]
        src.copy_(dev(np.stack(frames).reshape(case.frames, h, w, case.cn)))
    for path in paths_of(case):
        set_path(monkeypatch, path)
        if case.frames == 1:
            got = [to_host(device_resize(cvb, case, src))]
        else:
            fill = U8_FILL if case.dtype == "u8" else F32_FILL
            dbig = torch.full((case.frames, dh + 3, dw, case.cn), fill, dtype=tdt, device="cuda")
            device_resize(cvb, case, src, dst=dbig[:, :dh])
            out = to_host(dbig)
            assert np.all(out[:, dh:] == out.dtype.type(fill)), "path %s, case %s: rows between the frames were written" % (path, case.id)
            got = list(out[:, :dh])
        for i in range(case.frames):
            assert_same(got[i], want[i], case, path, ", frame %d" % i if case.frames > 1 else "")


# ------------------------------------------------------------------------------------------------------------------- views
def strided(buf, offset, shape, pitch):
    """(h, w[, cn]) view of the 1-D tensor / array buf starting `offset` elements in, rows `pitch` elements apart"""
    h, w, cn = shape
    if not isinstance(buf, np.ndarray):
        import torch
        t = torch.as_strided(buf, (h, w, cn), (pitch, cn, 1), offset)
    else:
        t = np.lib.stride_tricks.as_strided(buf[offset:], (h, w, cn), (pitch * buf.itemsize, cn * buf.itemsize, buf.itemsize))
    return t if cn > 1 else t[:, :, 0]


def _viewed(c):
    if c.frames > 1 or c.src[0] * c.src[1] > 200000 or c.dsize[0] * c.dsize[1] > 200000:
        return False
    return c.group in ("pp", "nn", "a2", "ex", "am", "fx") or (c.group == "sx" and "-w2" not in c.id and "-res" not in c.id) or \
        (c.group == "lz" and "-w" in c.id) or (c.group == "ai" and c.dtype == "u8")


VIEWS = [c for c in rc.CASES if _viewed(c)]


@pytest.mark.parametrize("case", VIEWS, ids=lambda c: c.id)
def test_views(cvb, port, monkeypatch, case):
    """The case with the source and the destination as views into larger buffers.  Source: rows padded to a multiple of 16 bytes
    plus 32, starting 1, 3, 4 and 16 bytes into the allocation (float: 4 and 16) -- word loads and 32-bit gathers only where the start
    is a multiple of 4.  Destination: a pitch that is a multiple of 4 starting at the allocation (32-bit stores, and their tail) and one
    element in (8-bit: byte stores).  The buffer around a destination view is pre-filled and must come back unchanged."""
    import torch
    img = rc.frames_of(case)[0]
    want = rc.run(port, case, img)
    h, w = case.src
    dw, dh = case.dsize
    u8 = case.dtype == "u8"
    esz = 1 if u8 else 4
    tdt, ndt = (torch.uint8, np.uint8) if u8 else (torch.float32, np.float32)
    spitch = ((w * case.cn * esz + 15) // 16 * 16 + 32) // esz
    gen = torch.Generator(device="cuda").manual_seed(5)
    for off in ((1, 3, 4, 16) if u8 else (4, 16)):              # bytes
        sbuf = torch.randint(0, 200, (h * spitch + 64,), generator=gen, device="cuda").to(tdt)
        src = strided(sbuf, off // esz, (h, w, case.cn), spitch)
        src.copy_(dev(img))
        aligned = off % 4 == 0
        for path in paths_of(case):
            set_path(monkeypatch, path)
            assert_same(to_host(device_resize(cvb, case, src)), want, case, path, ", source view %d bytes in, pitch %d" % (off, spitch * esz),
                        src_aligned=aligned)
    src = dev(img)
    fill = U8_FILL if u8 else F32_FILL
    dpitch = ((dw * case.cn * esz + 3) // 4 * 4 + 8) // esz
    for off in ((0, 1) if u8 else (0, 4)):                       # bytes
        expect = np.full(dh * dpitch + 64, fill, ndt)
        strided(expect, off // esz, (dh, dw, case.cn), dpitch)[...] = want
        for path in paths_of(case):
            set_path(monkeypatch, path)
            dbuf = torch.full((dh * dpitch + 64,), fill, dtype=tdt, device="cuda")
            dst = strided(dbuf, off // esz, (dh, dw, case.cn), dpitch)
            device_resize(cvb, case, src, dst=dst)
            what = ", destination view %d bytes in, pitch %d" % (off, dpitch * esz)
            assert_same(to_host(dst), want, case, path, what, dst_aligned=off % 4 == 0)
            assert rc.same(to_host(dbuf), expect), "path %s, case %s%s: bytes outside the view were written" % (path, case.id, what)


# ------------------------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("case", rc.REFUSALS, ids=lambda c: c.id)
def test_refusals(cvb, case):
    """rows >= 65536, NEAREST_EXACT with 32768 or more columns or rows, explicit 0.5 on odd sizes (the reference's partial last
    windows are not built) and explicit scales for interpolations that take their scale from the sizes: NOT_IMPLEMENTED, the
    destination untouched"""
    import torch
    h, w = case.src
    dw, dh = case.dsize
    tdt = torch.uint8 if case.dtype == "u8" else torch.float32
    src = torch.zeros((h, w, case.cn), dtype=tdt, device="cuda")
    dst = torch.full((dh, dw, case.cn), 3, dtype=tdt, device="cuda")
    with pytest.raises(C.NotImplementedOnDevice):
        device_resize(cvb, case, src, dst=dst)
    assert np.all(to_host(dst) == 3), "case %s: the destination of a refused call was written" % case.id


# ------------------------------------------------------------------------------------------------- which kernel a case runs on
_TARG = {"unsigned char": "u8", "float": "f32", "true": True, "false": False}


def _targs(s):
    return tuple(_TARG[a] if a in _TARG else int(a) for a in (x.strip() for x in s.split(",")))


def _mangled_targs(s):
    out = []
    for m in re.finditer(r"Li(\d+)E|Lb([01])E|(?<=[IE])([hf])", s):
        out.append(int(m.group(1)) if m.group(1) else bool(int(m.group(2))) if m.group(2) else ("u8" if m.group(3) == "h" else "f32"))
    return tuple(out)


def resize_kernels(trace):
    """[(kernel, template arguments, grid)] of the resize kernels (not the table builder) in a torch.profiler chrome trace, in launch order"""
    out = []
    for e in sorted((e for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"]):
        name = e["name"]
        d = re.search(r"(resize_\w+_kernel)<([^>]*)>", name)
        g = re.search(r"\d+(resize_\w+_kernel)(I.*?EE)", name)
        if d:
            k, args = d.group(1), _targs(d.group(2))
        elif g:
            k, args = g.group(1), _mangled_targs(g.group(2))
        else:
            continue
        if k != "resize_tab_kernel":
            out.append((k, args, tuple(e.get("args", {}).get("grid", ()))))
    return out


def kernel_runs():
    """[(case, path)] test_predicted_kernel_runs launches: every case that runs a kernel (default dispatch), and the NEAREST and
    LANCZOS4 switches"""
    todo = [(c, None) for c in rc.CASES if rc.predict(c).kernel != "copy"]
    todo += [(c, ("nn", p)) for c in rc.CASES if c.group == "nn" for p in ("v1", "walk")]
    todo += [(c, ("lz", "v1")) for c in rc.CASES if c.group == "lz" and c.dtype == "u8" and "-dh" in c.id]
    return todo


def capture_kernel_runs(trace):
    """launch kernel_runs() under torch.profiler and write its chrome trace to `trace` (run by test_predicted_kernel_runs in a process
    of its own)"""
    import os
    import torch
    from torch.profiler import ProfilerActivity, profile
    C.init(0)
    todo = kernel_runs()
    srcs = []
    for case, _ in todo:
        frames = rc.frames_of(case)
        srcs.append(dev(frames[0]) if case.frames == 1 else dev(np.stack(frames).reshape((case.frames,) + case.src + (case.cn,))))
    torch.cuda.synchronize()
    # one capture for all launches; the profiler now and then loses the first kernel record after it starts, so a few launches that
    # are not looked at come first and the records are counted from the end
    lead = 4
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for (case, path), src in zip([todo[0]] * lead + todo, [srcs[0]] * lead + srcs):
            for v in ENV.values():
                os.environ.pop(v, None)
            if path is not None:
                os.environ[ENV[path[0]]] = path[1]
            device_resize(C, case, src)
            if lead:
                torch.cuda.synchronize()
                lead -= 1
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(trace))


def test_predicted_kernel_runs(cvb, tmp_path):
    """resize_cases.predict() against the kernels that run, for every case that launches one (default dispatch) and for the NEAREST
    and LANCZOS4 switches: kernel, template arguments, and for resize_sep_u8_kernel and resize_lanczos4_sep_kernel a grid of
    ceil(dh / DH) row blocks.  Every kernel the table aims at runs, every DH of both tiled kernels among them.
    The capture (about 600 launches) runs in a child process: in the process of the suite, kernel records went missing from the
    short captures of later tests after it."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    trace = tmp_path / "trace.json"
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_resize_exact_edges as t; t.capture_kernel_runs(%r)" % (
        here, os.path.dirname(here), str(trace))
    env = {k: v for k, v in os.environ.items() if k not in ENV.values()}
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, "the capture process failed:\n%s" % r.stderr[-4000:]
    todo = kernel_runs()
    ran = resize_kernels(trace)
    assert len(todo) <= len(ran) <= len(todo) + 4, "%d resize kernels recorded for %d calls" % (len(ran), len(todo) + 4)
    ran = ran[-len(todo):]
    seen, dhs = set(), set()
    for (case, path), (kernel, args, grid) in zip(todo, ran):
        want = rc.predict(case, path)
        assert (kernel, args) == (want.kernel, want.args), "case %s path %s: predicted %s%s, ran %s%s" % (case.id, path, want.kernel, want.args, kernel, args)
        seen.add((kernel, args))
        if want.DH:
            assert grid[1] == -(-case.dsize[1] // want.DH), "case %s: %s grid %s, DH = %d" % (case.id, kernel, grid, want.DH)
            dhs.add((kernel, want.DH))
    for T in ("u8", "f32"):
        for cn in (1, 3, 4):
            for k in ("resize_linear_kernel", "resize_cubic_kernel", "resize_area_int_kernel", "resize_area_kernel", "resize_lanczos4_kernel"):
                assert (k, (T, cn)) in seen, (k, T, cn)
    for cn in (1, 3, 4):
        for k in ("resize_area2_u8_kernel", "resize_area2_f32_kernel", "resize_linear_exact_kernel", "resize_nn_walk_kernel", "resize_lanczos4_sep_kernel"):
            assert (k, (cn,)) in seen, (k, cn)
        assert ("resize_sep_u8_kernel", (cn, False)) in seen and ("resize_sep_u8_kernel", (cn, True)) in seen
    for pix in (1, 3, 4, 12, 16):
        assert ("resize_nn_kernel", (pix,)) in seen and ("resize_nn_exact_kernel", (pix,)) in seen
    assert {d for k, d in dhs if k == "resize_sep_u8_kernel"} == {64, 48, 32, 24, 16, 8, 4}
    assert {d for k, d in dhs if k == "resize_lanczos4_sep_kernel"} == {32, 16, 8, 4}
