"""Helpers for the -m gpu parity tests: they drive the CUDA path through the C-ABI (ctypes) with torch
tensors as device buffers and return numpy arrays for comparison with the oracle."""
import ctypes as C

import numpy as np

from dali_b200 import capi


def _torch():
    import torch
    return torch


def to_dev(arrs):
    torch = _torch()
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


def cmn(imgs, anchors, crops, mirrors, mean, inv_std, out_dtype=np.float32, layout="CHW", out_channels=None, fill=None, plan=None):
    torch = _torch()
    n = len(imgs)
    oc = out_channels or imgs[0].shape[2]
    samples = (capi.CmnSample * n)()
    for i, im in enumerate(imgs):
        s = samples[i]
        s.in_h, s.in_w, s.channels = im.shape
        s.anchor_y, s.anchor_x = anchors[i]
        s.crop_h, s.crop_w = crops[i]
        s.mirror = int(mirrors[i])
        s.mean[:] = list(capi.np_f32(mean, 4)); s.inv_std[:] = list(capi.np_f32(inv_std, 4))
        if np.asarray(mean).size < 4:
            for c in range(np.asarray(mean).size, 4):
                s.mean[c] = 0.0; s.inv_std[c] = 1.0
        s.fill[:] = list(capi.np_f32(fill, 4))
    plan = plan or capi.Plan("Cmn", max(n, 1))
    dt = capi.FLOAT if np.dtype(out_dtype) == np.float32 else capi.FLOAT16
    capi.check(capi.lib().dalib200CmnPlanSetup(plan.handle, n, samples, dt, capi.LAYOUT_CHW if layout == "CHW" else capi.LAYOUT_HWC, oc))
    din = to_dev(imgs)
    tdt = torch.float32 if dt == capi.FLOAT else torch.float16
    outs = [torch.empty((oc, c[0], c[1]) if layout == "CHW" else (c[0], c[1], oc), dtype=tdt, device="cuda") for c in crops]
    capi.check(capi.lib().dalib200CmnLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


def fill_resample_sample(s, shape, out_hw, min_filter, mag_filter, roi):
    s.in_h, s.in_w, s.channels = shape
    s.out_h, s.out_w = out_hw
    def pair(f):
        return [capi.make_filter(f[0]), capi.make_filter(f[1])] if isinstance(f, list) else [capi.make_filter(f), capi.make_filter(f)]
    mn, mg = pair(min_filter), pair(mag_filter)
    for d in range(2):
        s.min_filter[d] = mn[d]; s.mag_filter[d] = mg[d]
        s.use_roi[d] = 0
        if roi is not None and roi[0][d] is not None:
            s.use_roi[d] = 1; s.roi_start[d] = roi[0][d]; s.roi_end[d] = roi[1][d]


def resample(imgs, out_hws, min_filter=(capi.FILTER_LINEAR, 1, 0.0), mag_filter=(capi.FILTER_LINEAR, 1, 0.0), out_dtype=None,
             rois=None, want_order=False, plan=None, want_path=False):
    torch = _torch()
    n = len(imgs)
    samples = (capi.ResampleSample * n)()
    for i, im in enumerate(imgs):
        fill_resample_sample(samples[i], im.shape, out_hws[i], min_filter, mag_filter, rois[i] if rois else None)
    in_dt = capi.UINT8 if imgs[0].dtype == np.uint8 else capi.FLOAT
    out_dtype = np.dtype(out_dtype or imgs[0].dtype)
    out_dt = capi.UINT8 if out_dtype == np.uint8 else capi.FLOAT
    plan = plan or capi.Plan("Resample", max(n, 1))
    capi.check(capi.lib().dalib200ResamplePlanSetup(plan.handle, n, samples, in_dt, out_dt))
    din = to_dev(imgs)
    outs = [torch.empty((hw[0], hw[1], im.shape[2]), dtype=torch.uint8 if out_dt == capi.UINT8 else torch.float32, device="cuda")
            for hw, im in zip(out_hws, imgs)]
    capi.check(capi.lib().dalib200ResampleLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    res = [o.cpu().numpy() for o in outs]
    if want_path:
        return res, [capi.lib().dalib200ResamplePlanGetPath(plan.handle, i) for i in range(n)]
    if want_order:
        return res, [capi.lib().dalib200ResamplePlanGetOrder(plan.handle, i) for i in range(n)]
    return res


def synth_image(h, w, seed):
    """SURVEY.md 8(d) C2 recipe: bicubic-upsampled low-frequency noise + sigma=5 gaussian noise."""
    import cv2
    r = np.random.default_rng(seed)
    lo = r.uniform(0, 255, (max(2, h // 32), max(2, w // 32), 3)).astype(np.float32)
    img = cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC) + r.normal(0, 5, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def random_crop_window(seed, sample_idx, H, W, area=(0.08, 1.0), aspect=(3 / 4, 4 / 3), num_attempts=10, ncalls=1):
    """(anchor_y, anchor_x, h, w) of the ncalls-th window the library's random crop generator draws for sample_idx: the one that
    decoders.image_random_crop / random_resized_crop with this seed use in their ncalls-th iteration (host code only; the generator
    is pinned to the reference's by tests/test_host_cpu.py where oracle/_ref exists)."""
    from dali_b200 import backend
    w = (C.c_int * (4 * ncalls))()
    assert backend.lib().dalihTestRandomCrop(C.c_int64(seed), int(sample_idx), int(H), int(W), C.c_float(aspect[0]), C.c_float(aspect[1]),
                                             C.c_float(area[0]), C.c_float(area[1]), int(num_attempts), int(ncalls), w) == 0
    return tuple(w[4 * (ncalls - 1):4 * ncalls])


def jpeg_decode(streams, output_type=capi.RGB, fancy=True, plan=None, want_coefs=False):
    torch = _torch()
    n = len(streams)
    bufs = [np.frombuffer(bytes(s), np.uint8) for s in streams]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * n)(*[b.size for b in bufs])
    plan = plan or capi.Plan("Jpeg", max(n, 1))
    capi.check(capi.lib().dalib200JpegPlanSetup(plan.handle, n, ptrs, lens, output_type, int(fancy)))
    outs, infos = [], []
    for i in range(n):
        info = capi.JpegInfo()
        capi.check(capi.lib().dalib200JpegPlanGetInfo(plan.handle, i, C.byref(info)))
        infos.append(info)
        ch = 1 if output_type == capi.GRAY else 3
        outs.append(torch.empty((info.height, info.width, ch), dtype=torch.uint8, device="cuda"))
    capi.check(capi.lib().dalib200JpegUpload(plan.handle, capi.stream_handle()))
    capi.check(capi.lib().dalib200JpegLaunch(plan.handle, capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    status = (C.c_int32 * n)()
    capi.check(capi.lib().dalib200JpegGetStatus(plan.handle, status))
    res = [o.cpu().numpy() for o in outs]
    if want_coefs:
        return res, list(status), plan
    return res, list(status)


def jpeg_decode_ex(streams, output_type=capi.RGB, fancy=True, dtype=capi.UINT8, adjust_orientation=True, rois=None, plan=None, pinned=False,
                   want_upload_path=False):
    """dalib200JpegPlanSetupEx: rois[i] = None | (x0, y0, x1, y1) in output (oriented) coordinates.  pinned=True: the streams live in
    page-locked memory and are declared stable (dalib200JpegPlanSetSourceStable) -> no host repack."""
    torch = _torch()
    n = len(streams)
    bufs = [np.frombuffer(bytes(s), np.uint8) for s in streams]
    if pinned:
        arena = capi.pinned_empty(sum((b.size + 63) & ~63 for b in bufs) + 64)
        off, pb = 0, []
        for b in bufs:
            v = arena[off:off + b.size]
            v[:] = b
            pb.append(v)
            off += (b.size + 63) & ~63
        bufs = pb
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * n)(*[b.size for b in bufs])
    plan = plan or capi.Plan("Jpeg", max(n, 1))
    prm = capi.JpegParams(output_type, int(fancy), dtype, int(adjust_orientation))
    capi.check(capi.lib().dalib200JpegPlanSetSourceStable(plan.handle, int(pinned)))
    cr = None
    if rois is not None:
        cr = (capi.JpegRoi * n)()
        for i, r in enumerate(rois):
            if r is not None:
                cr[i].use_roi = 1
                cr[i].x0, cr[i].y0, cr[i].x1, cr[i].y1 = [int(v) for v in r]
    capi.check(capi.lib().dalib200JpegPlanSetupEx(plan.handle, n, ptrs, lens, C.byref(prm), cr))
    outs = []
    for i in range(n):
        hwc = (C.c_int32 * 3)()
        capi.check(capi.lib().dalib200JpegPlanGetOutputShape(plan.handle, i, hwc))
        outs.append(torch.empty(tuple(hwc), dtype=torch.uint8 if dtype == capi.UINT8 else torch.float32, device="cuda"))
    capi.check(capi.lib().dalib200JpegUpload(plan.handle, capi.stream_handle()))
    capi.check(capi.lib().dalib200JpegLaunch(plan.handle, capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    status = (C.c_int32 * n)()
    capi.check(capi.lib().dalib200JpegGetStatus(plan.handle, status))
    if want_upload_path:
        return [o.cpu().numpy() for o in outs], list(status), int(capi.lib().dalib200JpegPlanLastUploadDirect(plan.handle))
    return [o.cpu().numpy() for o in outs], list(status)


def jpeg_coefs(plan, sample, count):
    out = np.empty(count, np.int16)
    capi.check(capi.lib().dalib200JpegDebugGetCoefficients(plan.handle, sample, out.ctypes.data_as(C.c_void_p), C.c_size_t(count)))
    return out


def warp_affine(imgs, mats, out_hws=None, interp=1, fill=None, out_dtype=np.uint8, contiguous=False, want_path=False):
    """contiguous=True: the inputs are slices of ONE device allocation (like the frames of an FHWC batch) -> the tensor-map TMA
    kernel can take them; want_path=True also returns dalib200WarpPlanGetPath."""
    torch = _torch()
    n = len(imgs)
    samples = (capi.WarpSample * n)()
    for i, im in enumerate(imgs):
        s = samples[i]
        s.in_h, s.in_w, s.channels = im.shape
        s.out_h, s.out_w = out_hws[i] if out_hws else im.shape[:2]
        s.matrix[:] = [float(v) for v in np.asarray(mats[i], np.float32).reshape(6)]
    plan = capi.Plan("Warp", max(n, 1))
    odt = capi.UINT8 if np.dtype(out_dtype) == np.uint8 else capi.FLOAT
    capi.check(capi.lib().dalib200WarpPlanSetup(plan.handle, n, samples, int(interp), int(fill is not None), C.c_float(fill or 0.0), odt))
    if contiguous:
        whole = torch.from_numpy(np.stack(imgs)).cuda()
        din = [whole[i] for i in range(n)]
    else:
        din = to_dev(imgs)
    outs = [torch.empty((samples[i].out_h, samples[i].out_w, imgs[i].shape[2]), dtype=torch.uint8 if odt == capi.UINT8 else torch.float32,
                        device="cuda") for i in range(n)]
    capi.check(capi.lib().dalib200WarpLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    res = [o.cpu().numpy() for o in outs]
    return (res, capi.lib().dalib200WarpPlanGetPath(plan.handle)) if want_path else res


def color_twist_matrix(hue=0.0, saturation=1.0, value=1.0, brightness=1.0, contrast=1.0, half_range=128.0):
    M, T = np.empty(9, np.float32), np.empty(3, np.float32)
    capi.lib().dalib200ColorTwistMatrix(C.c_float(hue), C.c_float(saturation), C.c_float(value), C.c_float(brightness),
                                       C.c_float(contrast), C.c_float(half_range), M.ctypes.data_as(C.c_void_p), T.ctypes.data_as(C.c_void_p))
    return M.reshape(3, 3), T


def linear_transform(imgs, mats, offs, out_dtype=np.uint8):
    torch = _torch()
    n = len(imgs)
    samples = (capi.ColorSample * n)()
    for i, im in enumerate(imgs):
        samples[i].num_pixels = im.size // 3
        samples[i].matrix[:] = [float(v) for v in np.asarray(mats[i], np.float32).reshape(9)]
        samples[i].offset[:] = [float(v) for v in np.asarray(offs[i], np.float32).reshape(3)]
    plan = capi.Plan("Pointwise", max(n, 1))
    odt = capi.UINT8 if np.dtype(out_dtype) == np.uint8 else capi.FLOAT
    capi.check(capi.lib().dalib200LinearTransformSetup(plan.handle, n, samples, odt))
    din = to_dev(imgs)
    outs = [torch.empty(im.shape, dtype=torch.uint8 if odt == capi.UINT8 else torch.float32, device="cuda") for im in imgs]
    capi.check(capi.lib().dalib200PointwiseLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


def csc(imgs, in_type, out_type):
    torch = _torch()
    n = len(imgs)
    ic = 1 if in_type == capi.GRAY else 3
    oc = 1 if out_type == capi.GRAY else 3
    npx = (C.c_int64 * n)(*[im.size // ic for im in imgs])
    plan = capi.Plan("Pointwise", max(n, 1))
    capi.check(capi.lib().dalib200ColorSpaceSetup(plan.handle, n, npx, in_type, out_type))
    din = to_dev(imgs)
    outs = [torch.empty(im.shape[:-1] + (oc,), dtype=torch.uint8, device="cuda") for im in imgs]
    capi.check(capi.lib().dalib200PointwiseLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


def spectrogram(sigs, nfft=None, window_length=512, window_step=256, power=2, center=True, reflect=True, layout="ft", window_fn=None,
                plan=None):
    """plan: an existing capi.Plan("Spectrogram", ...) to set up again (default: a fresh one)."""
    torch = _torch()
    n = len(sigs)
    args = capi.SpectrogramArgs(nfft or window_length, window_length, window_step, power, int(center), int(reflect), int(layout == "ft"))
    lens = (C.c_int64 * n)(*[int(s.size) for s in sigs])
    if plan is None:
        plan = capi.Plan("Spectrogram", max(n, 1))
    wf = None
    if window_fn is not None:
        wfa = np.ascontiguousarray(window_fn, np.float32)
        wf = wfa.ctypes.data_as(C.c_void_p)
    capi.check(capi.lib().dalib200SpectrogramPlanSetup(plan.handle, C.byref(args), wf, n, lens))
    nbin = args.nfft // 2 + 1
    din = to_dev([np.ascontiguousarray(s, np.float32) for s in sigs])
    outs = []
    for i in range(n):
        nw = capi.lib().dalib200SpectrogramNumWindows(plan.handle, i)
        outs.append(torch.empty((nbin, nw) if layout == "ft" else (nw, nbin), dtype=torch.float32, device="cuda"))
    capi.check(capi.lib().dalib200SpectrogramLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


def mel_filter_bank(specs, nfilter=128, sample_rate=44100.0, freq_low=0.0, freq_high=0.0, mel_formula="slaney", normalize=True,
                    tensor_cores=False):
    torch = _torch()
    n = len(specs)
    args = capi.MelArgs(nfilter, sample_rate, freq_low, freq_high, int(mel_formula == "htk"), int(bool(normalize)))
    nwin = (C.c_int64 * n)(*[int(s.shape[1]) for s in specs])
    plan = capi.Plan("Mel", max(n, 1))
    capi.check(capi.lib().dalib200MelPlanSetTensorCores(plan.handle, int(tensor_cores)))
    capi.check(capi.lib().dalib200MelPlanSetup(plan.handle, C.byref(args), int(specs[0].shape[0]), n, nwin))
    din = to_dev([np.ascontiguousarray(s, np.float32) for s in specs])
    outs = [torch.empty((nfilter, s.shape[1]), dtype=torch.float32, device="cuda") for s in specs]
    capi.check(capi.lib().dalib200MelLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


def spectrogram_mel_fused(sigs, nfilter=128, sample_rate=16000.0, freq_high=8000.0, keep_spectrogram=True, **spec_kw):
    """dalib200SpectrogramMelLaunch: (spectrograms or None, mel outputs); the spectrogram arguments are those of `spectrogram`."""
    torch = _torch()
    n = len(sigs)
    wl = spec_kw.get("window_length", 512)
    nfft = spec_kw.get("nfft") or wl
    args = capi.SpectrogramArgs(nfft, wl, spec_kw.get("window_step", 256), spec_kw.get("power", 2), int(spec_kw.get("center", True)),
                                int(spec_kw.get("reflect", True)), 1)
    lens = (C.c_int64 * n)(*[int(s.size) for s in sigs])
    sp = capi.Plan("Spectrogram", max(n, 1))
    capi.check(capi.lib().dalib200SpectrogramPlanSetup(sp.handle, C.byref(args), None, n, lens))
    nbin = nfft // 2 + 1
    nws = [int(capi.lib().dalib200SpectrogramNumWindows(sp.handle, i)) for i in range(n)]
    margs = capi.MelArgs(nfilter, sample_rate, 0.0, freq_high, 0, 1)
    mp = capi.Plan("Mel", max(n, 1))
    capi.check(capi.lib().dalib200MelPlanSetup(mp.handle, C.byref(margs), nbin, n, (C.c_int64 * n)(*nws)))
    assert capi.lib().dalib200SpectrogramMelSupported(sp.handle, mp.handle) == 1
    din = to_dev([np.ascontiguousarray(s, np.float32) for s in sigs])
    specs = [torch.zeros((nbin, nw), dtype=torch.float32, device="cuda") for nw in nws]
    mels = [torch.empty((nfilter, nw), dtype=torch.float32, device="cuda") for nw in nws]
    capi.check(capi.lib().dalib200SpectrogramMelLaunch(sp.handle, mp.handle, capi.ptr_array(din), capi.ptr_array(specs) if keep_spectrogram else None,
                                                       capi.ptr_array(mels), capi.stream_handle()))
    torch.cuda.synchronize()
    return ([o.cpu().numpy() for o in specs] if keep_spectrogram else None), [o.cpu().numpy() for o in mels]


def resample3d(vols, out_dhws, min_filter, mag_filter, out_dtype=None, rois=None, want_order=False, plan=None):
    """DHWC volumes through dalib200Resample3D* (per-axis filter lists in shape order [z, y, x])."""
    import ctypes as C
    torch = _torch()
    n = len(vols)
    samples = (capi.Resample3DSample * n)()
    for i, v in enumerate(vols):
        s, roi = samples[i], rois[i] if rois else None
        for d in range(3):
            s.in_shape[d], s.out_shape[d] = int(v.shape[d]), int(out_dhws[i][d])
            s.min_filter[d] = capi.FilterDesc(*[t(x) for t, x in zip((int, int, float), min_filter[d])])
            s.mag_filter[d] = capi.FilterDesc(*[t(x) for t, x in zip((int, int, float), mag_filter[d])])
            if roi is not None and roi[0][d] is not None:
                s.use_roi[d], s.roi_start[d], s.roi_end[d] = 1, roi[0][d], roi[1][d]
        s.channels = int(v.shape[3])
    in_dt = capi.UINT8 if vols[0].dtype == np.uint8 else capi.FLOAT
    out_dtype = np.dtype(out_dtype or vols[0].dtype)
    out_dt = capi.UINT8 if out_dtype == np.uint8 else capi.FLOAT
    plan = plan or capi.Plan("Resample3D", max(n, 1))
    capi.check(capi.lib().dalib200Resample3DPlanSetup(plan.handle, n, samples, in_dt, out_dt))
    din = to_dev(vols)
    outs = [torch.empty(tuple(int(x) for x in o) + (v.shape[3],), dtype=torch.uint8 if out_dt == capi.UINT8 else torch.float32, device="cuda")
            for o, v in zip(out_dhws, vols)]
    capi.check(capi.lib().dalib200Resample3DLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    res = [o.cpu().numpy() for o in outs]
    if want_order:
        orders = []
        for i in range(n):
            o = (C.c_int32 * 3)()
            capi.check(capi.lib().dalib200Resample3DPlanGetOrder(plan.handle, i, o))
            orders.append(list(o))
        return res, orders
    return res
