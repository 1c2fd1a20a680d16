"""warpAffine / warpPerspective / remap on the device held to the C port (oracle/port/port_geometry.c, warp_impl) bit for bit, over the
table of tests/warp_cases.py.  tests/test_warp_port.py holds the port to the reference over the same table, so nothing here needs
the reference and nothing skips.

Four kernels do the warps' arithmetic with different work splits (opencv_b200/csrc/warp.cu): warp_kernel (direct gather),
warp_tile_kernel (64x16 tiles, staged footprint), warp_tile4_kernel (8-bit LINEAR / CUBIC, 128x32 tiles, 4 pixels per thread) and
warp_nn4_kernel (8-bit NEAREST, the same tables without staging).  Every case runs through the default dispatch, through
B200CV_WARP_PATH=direct and, for LINEAR / CUBIC, through B200CV_WARP_PATH=tile64, which is how the 8-bit instantiations of
warp_tile_kernel are reached at all at these sizes.  warp_cases.predict() restates the dispatch; test_predicted_kernel_runs checks it,
template arguments included, against the kernels torch.profiler sees.

A failure names the forced path, the case, the first differing pixel and where it sits: its 128-column tile, its projective
column block and its place in a thread's 4-pixel group.
"""
import json
import re

import numpy as np
import pytest

import opencv_b200 as C
import warp_cases as wc

pytestmark = pytest.mark.gpu

U8_FILL, F32_FILL = 0xA5, -777.25


def paths_of(case):
    return (None, "direct") if case.flags & 7 == wc.NEAREST else (None, "direct", "tile64")


def set_path(monkeypatch, path):
    if path is None:
        monkeypatch.delenv("B200CV_WARP_PATH", raising=False)
    else:
        monkeypatch.setenv("B200CV_WARP_PATH", path)


def device_warp(cvb, case, src, dst=None):
    fn = cvb.warpAffine if case.op == "affine" else cvb.warpPerspective
    return fn(src, wc.matrix(case), case.dsize, case.flags, case.border, case.bval, dst=dst)


def to_host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def assert_same(got, want, case, path, what=""):
    """got == want for one frame, (h, w) or (h, w, cn)"""
    got = np.asarray(got).reshape(want.shape)
    if np.array_equal(got, want):
        return
    bad = np.argwhere(got != want)
    y, x = int(bad[0][0]), int(bad[0][1])
    bw0 = wc.block_width(case)
    where = "128-column tile %d, 64-column tile %d, pixel %d of its 4-pixel group" % (x // 128, x // 64, x % 4)
    if case.op == "perspective":
        where += ", column block %d of width bw0 = %d (offset %d)" % (x // bw0, bw0, x % bw0)
    raise AssertionError("path %s (%s), case %s%s: %d of %d elements differ, first at x = %d, y = %d: got %s want %s; %s" % (
        path or "default", wc.predict(case, path), case.id, what, len(bad), got.size, x, y, got[y, x], want[y, x], where))


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---------------------------------------------------------------------------------------------------------------- the whole table
@pytest.mark.parametrize("case", wc.CASES, ids=lambda c: c.id)
def test_kernels_vs_port(cvb, port, monkeypatch, case):
    import torch
    frames = wc.frames_of(case)
    want = [wc.run(port, case, f) for f in frames]
    dw, dh = case.dsize
    if case.frames == 1:
        src = dev(frames[0])
    else:
        # a batch whose frame stride is larger than a frame: (N, h + 2, w, cn)[:, :h], and (N, dh + 3, dw, cn)[:, :dh] for the destination
        h, w = case.src
        big = torch.full((case.frames, h + 2, w, case.cn), 99, dtype=torch.uint8 if case.dtype == "u8" else torch.float32, device="cuda")
        src = big[:, :h]
        src.copy_(dev(np.stack(frames).reshape(case.frames, h, w, case.cn)))
    for path in paths_of(case):
        set_path(monkeypatch, path)
        if case.frames == 1:
            got = [to_host(device_warp(cvb, case, src))]
        else:
            fill = U8_FILL if case.dtype == "u8" else F32_FILL
            dbig = torch.full((case.frames, dh + 3, dw, case.cn), fill, dtype=src.dtype, device="cuda")
            device_warp(cvb, case, src, dst=dbig[:, :dh])
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


ALIGN = [c for c in wc.CASES if c.group == "al"]


@pytest.mark.parametrize("case", ALIGN, ids=lambda c: c.id)
def test_views(cvb, port, monkeypatch, case):
    """The `al` cases again with the source and the destination as views into larger buffers.  Source: rows padded to a multiple of
    16 bytes plus 32, starting 1, 3, 4 and 16 bytes into the allocation -- only the last keeps the 16-byte vector loads.  Destination:
    a pitch that is a multiple of 4 starting at the allocation (32-bit stores, and their tail for widths 4k + 1 .. 4k + 3) and one
    byte in (byte stores).  The buffer around a destination view is pre-filled and must come back unchanged."""
    import torch
    img = wc.frames_of(case)[0]
    want = wc.run(port, case, img)
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
        assert (src.data_ptr() % 16 == 0) == (off == 16)
        for path in paths_of(case):
            set_path(monkeypatch, path)
            assert_same(to_host(device_warp(cvb, case, src)), want, case, path, ", source view %d bytes in, pitch %d" % (off, spitch * esz))
    src = dev(img)
    fill = U8_FILL if u8 else F32_FILL
    dpitch = ((dw * case.cn * esz + 3) // 4 * 4 + 8) // esz
    for off in ((0, 1) if u8 else (0, 1 * 4)):                   # bytes
        expect = np.full(dh * dpitch + 64, fill, ndt)
        strided(expect, off // esz, (dh, dw, case.cn), dpitch)[...] = want
        for path in paths_of(case):
            set_path(monkeypatch, path)
            dbuf = torch.full((dh * dpitch + 64,), fill, dtype=tdt, device="cuda")
            dst = strided(dbuf, off // esz, (dh, dw, case.cn), dpitch)
            device_warp(cvb, case, src, dst=dst)
            what = ", destination view %d bytes in, pitch %d" % (off, dpitch * esz)
            assert_same(to_host(dst), want, case, path, what)
            assert np.array_equal(to_host(dbuf), expect), "path %s, case %s%s: bytes outside the view were written" % (path, case.id, what)


# ------------------------------------------------------------------------------------------------- which kernel a case runs on
def warp_kernels(prof, tmp_path):
    """[(kernel, (type, channels, interpolation) | None)] of the warp kernels in a torch.profiler capture, in launch order"""
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    out = []
    for e in sorted((e for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"]):
        m = re.search(r"warp_(?:tile4_|tile_|nn4_)?kernel", e["name"])
        if not m:
            continue
        inst = None
        d = re.search(r"warp_tile_kernel<([^>]*)>", e["name"])          # demangled: warp_tile_kernel<unsigned char, 3, 1>
        g = re.search(r"warp_tile_kernelI([hf])Li(\d)ELi(\d)E", e["name"])  # mangled
        if d:
            n = re.findall(r"\d+", d.group(1))
            inst = ("f32" if "float" in d.group(1) else "u8", int(n[-2]), int(n[-1]))
        elif g:
            inst = ("f32" if g.group(1) == "f" else "u8", int(g.group(2)), int(g.group(3)))
        out.append((m.group(0), inst))
    return out


def test_predicted_kernel_runs(cvb, monkeypatch, tmp_path):
    """warp_cases.predict() against the kernels that run: the footprint cases land on the kernel the table says (so they straddle
    the 96 KB decisions), widths 42 | 43 straddle `blocks_ok`, all four kernels run batches, and the `t64` cases reach each of the
    twelve (type, channels, LINEAR | CUBIC) instantiations of warp_tile_kernel -- the 8-bit ones through B200CV_WARP_PATH=tile64"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    todo = [(c, None) for c in wc.CASES if c.group == "fp" and c.flags & 7 != wc.NEAREST]
    todo += [(c, None) for c in wc.CASES if c.group == "bt"]
    todo += [(wc.BY_ID["bww-w%d-u8c1-%s-strong" % (w, i)], None) for w in (42, 43) for i in ("nn", "lin")]
    todo += [(wc.BY_ID["bt-affine-u8c3-lin"], p) for p in ("direct", "tile64")]
    t64 = [c for c in wc.CASES if c.group == "t64" and c.id.startswith("t64-rot")]
    todo += [(c, "tile64" if c.dtype == "u8" else None) for c in t64]
    # One capture for all launches; every call launches one warp kernel.  The profiler now and then loses the first kernel record
    # after it starts (late in a long process more often than not), so a capture per launch is unreliable: a few launches that are not
    # looked at come first, and the records are counted from the end.
    srcs = []
    for case, _ in todo:
        frames = wc.frames_of(case)
        srcs.append(dev(frames[0]) if case.frames == 1 else dev(np.stack(frames).reshape((case.frames,) + case.src + (case.cn,))))
    torch.cuda.synchronize()
    lead = 4
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for (case, path), src in zip([todo[0]] * lead + todo, [srcs[0]] * lead + srcs):
            set_path(monkeypatch, path)
            device_warp(cvb, case, src)
            if lead:
                torch.cuda.synchronize()
                lead -= 1
        torch.cuda.synchronize()
    ran = warp_kernels(prof, tmp_path)
    assert len(todo) <= len(ran) <= len(todo) + 4, "%d warp kernels recorded for %d calls" % (len(ran), len(todo) + 4)
    ran = ran[-len(todo):]
    seen, insts, batch = set(), set(), set()
    for (case, path), (kernel, inst) in zip(todo, ran):
        want = wc.predict(case, path)
        assert kernel == want, "case %s path %s: predicted %s, ran %s %s" % (case.id, path, want, kernel, inst)
        seen.add(want)
        if case.frames > 1:
            batch.add(want)
        if want == "warp_tile_kernel":
            it = wc.LINEAR if case.flags & 7 == wc.AREA else case.flags & 7
            assert inst == (case.dtype, case.cn, it), "case %s: instantiation %s" % (case.id, inst)
            insts.add(inst)
    every = {"warp_kernel", "warp_tile_kernel", "warp_tile4_kernel", "warp_nn4_kernel"}
    assert seen == every and batch == every
    assert insts == {(t, cn, it) for t in ("u8", "f32") for cn in (1, 3, 4) for it in (wc.LINEAR, wc.CUBIC)}
    assert wc.predict(wc.BY_ID["bww-w42-u8c1-lin-strong"]) == "warp_tile_kernel" and wc.predict(wc.BY_ID["bww-w43-u8c1-lin-strong"]) == "warp_tile4_kernel"
    assert wc.predict(wc.BY_ID["bww-w42-u8c1-nn-strong"]) == "warp_kernel" and wc.predict(wc.BY_ID["bww-w43-u8c1-nn-strong"]) == "warp_nn4_kernel"


# ------------------------------------------------------------------------------------------------------------------- remap
@pytest.mark.parametrize("dtype,cn", wc.TYPES6)
def test_remap_fixed_point_without_fractions(cvb, port, dtype, cn):
    """cv::remap(CV_16SC2 map, no second map): NEAREST uses the coordinates as they are (imgwarp.cpp:1166); any other interpolation
    has no fractions to work with and is refused with B200CV_ERR_BAD_ARG (-2), the destination untouched"""
    case = wc.remap_case(dtype, cn)
    img = wc.frames_of(case)[0]
    xy = wc.fixed_maps()
    for border in wc.BORDERS:
        got = to_host(cvb.remap(dev(img), dev(xy), None, wc.NEAREST, border, wc.BV4))
        want = port.remap(img, xy, None, wc.NEAREST, border, wc.BV4)
        assert np.array_equal(got.reshape(want.shape), want), "remap fixed-point maps, %s border %d: first difference at %s" % (
            case.id, border, np.argwhere(got.reshape(want.shape) != want)[0])
    for interp in (wc.LINEAR, wc.CUBIC):
        dst = dev(np.full((30, 44) + img.shape[2:], 3, img.dtype))
        with pytest.raises(C.B200cvError, match=r"\(-2\)") as e:
            cvb.remap(dev(img), dev(xy), None, interp, wc.REPL, 0, dst=dst)
        assert not isinstance(e.value, C.NotImplementedOnDevice)
        assert np.all(to_host(dst) == 3)
