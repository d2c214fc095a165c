"""Host mirror of the reference's Undistort set-up (util/Undistort.cpp) for the Pinhole camera model — the one every calibration file the
reference ships uses (calib/KITTI/*.txt, calib/kitti_360.txt, calib/kitti_carla.txt).

This is calibration-load-time work (once per run), not the per-frame path: it produces what the reference's Undistort object holds after
readFromFile (:666-886) — the rectified camera matrix K and the remapX/remapY tables — which Context.setUndistort hands to the device
(sdv_set_undistort); the per-frame rectification itself (Undistort::undistort, :341-435) runs fused in the CUDA ingest kernel.

The arithmetic follows the reference's float / double mix operation by operation (makeOptimalK_crop :538-659, UndistortPinhole::distortCoordinates
:1127-1152, the "rounding resistant" pass :859-881), so the tables are bit-identical to the reference's (tests/test_undistort.py checks that
against the reference's own compiled Undistort).  numpy note: float32-array (op) python-float stays float32, so every double-precision step of the reference is spelled
with an explicit float64 round trip.
"""
from __future__ import annotations
import numpy as np

f32 = np.float32


def _f32_of_f64(x) -> np.float32:
    return np.float32(np.float64(x))


def _parse_floats(line: str) -> list:
    """std::istream_iterator<float> over one line: tokens read as float (strtof, correctly rounded) up to the first one that is not a number"""
    out = []
    for tok in line.split():
        try:
            d = float(tok)
        except ValueError:
            break
        f = np.float32(d)
        if np.float64(f) != d:                                                 # not exactly a float: round the decimal text once, as strtof does
            f = np.float32(_strtof(tok.encode(), None))
        out.append(f)
    return out


def _strtof(s, end):
    import ctypes
    fn = ctypes.CDLL(None).strtof; fn.restype = ctypes.c_float; fn.argtypes = [ctypes.c_char_p, ctypes.c_void_p]
    return fn(s, end)


class PhotometricUndistorter:
    """Host mirror of the reference's PhotometricUndistorter constructor (util/Undistort.cpp:20-143) and of what processFrame (:177-214) applies.

    gamma_text: the response file's text; its first line holds GDepth >= 256 values of the inverse response G, strictly increasing.  vignette: the
    vignette image as a (h, w) uint16 (readImageBW_16U) or uint8 (readImageBW_8U) array of the raw size, or None.  photometric_calibration: the
    reference's setting_photometricCalibration (2 by default; src/main.cpp modes 1 and 2 set 0).  Any failure leaves the object invalid: getG() is
    None, and processFrame falls back to factor*v, as in the reference."""

    def __init__(self, gamma_text: str | None, vignette, w: int, h: int, photometric_calibration: int = 2):
        self.w, self.h = int(w), int(h); self.photometric_calibration = int(photometric_calibration)
        self.valid = False; self.G = None; self.GDepth = 0; self.vignetteMap = None; self.vignetteMapInv = None
        if gamma_text is None:                                                 # `if (!f.good()) return;`
            return
        lines = gamma_text.splitlines()
        Gvec = _parse_floats(lines[0] if lines else "")
        self.GDepth = GDepth = len(Gvec)
        if GDepth < 256:
            return
        G = np.array(Gvec, np.float32)
        if np.any(G[1:] <= G[:-1]):                                            # "G invalid! it has to be strictly increasing"
            return
        mn, mx = G[0], G[GDepth - 1]
        G = (255.0 * (G - mn).astype(np.float64) / np.float64(mx - mn)).astype(np.float32)   # 255.0 * (G[i]-min) / (max-min): float difference, double rest
        if self.photometric_calibration == 0:
            G = (f32(255.0) * np.arange(GDepth, dtype=f32)) / f32(GDepth - 1)
        self.G = G
        if vignette is None:
            return
        v = np.asarray(vignette)
        if v.dtype not in (np.uint16, np.uint8) or v.shape != (self.h, self.w):
            return                                                             # "Invalid vignette image (size)"
        vf = v.astype(f32); maxV = f32(0)
        if v.size:
            maxV = max(f32(0), vf.max())
        self.vignetteMap = vf / maxV
        self.vignetteMapInv = f32(1.0) / self.vignetteMap
        self.valid = True

    def getG(self):
        """PhotometricUndistorter::getG(): the GDepth-entry G when valid, else None (FullSystem::setGammaFunction then keeps the identity)"""
        return self.G if self.valid else None

    @property
    def ingest_G(self):
        """the 256-entry response processFrame<unsigned char> applies to frames with exposure > 0, or None where it applies factor*v"""
        return self.G[:256].copy() if self.valid and self.photometric_calibration != 0 else None

    @property
    def ingest_vignetteMapInv(self):
        """the inverse vignette processFrame multiplies in (setting_photometricCalibration == 2 only), or None"""
        return self.vignetteMapInv if self.ingest_G is not None and self.photometric_calibration == 2 else None

    def processFrame(self, raw, exposure: float = 1.0, factor: float = 1.0):
        """PhotometricUndistorter::processFrame<unsigned char> on a raw (h, w) mono8 image (test / data-preparation helper)"""
        raw = np.asarray(raw, np.uint8); assert raw.shape == (self.h, self.w)
        if self.ingest_G is None or not exposure > 0:
            return f32(factor) * raw.astype(f32)
        out = self.G[raw.astype(np.int64)]
        if self.photometric_calibration == 2:
            out = out * self.vignetteMapInv
        return out.astype(f32)

    @staticmethod
    def from_files(gamma_path: str | None, vignette_path: str | None, w: int, h: int, photometric_calibration: int = 2) -> "PhotometricUndistorter":
        """the constructor's file reads: the response text, and the vignette as a binary PGM (8 or 16 bit)"""
        try:
            with open(gamma_path) as f:
                text = f.read()
        except (OSError, TypeError):
            text = None
        try:
            vig = read_pgm(vignette_path)
        except (OSError, TypeError, ValueError):
            vig = None
        return PhotometricUndistorter(text, vig, w, h, photometric_calibration)


def read_pgm(path: str):
    """binary PGM (P5): uint8 for maxval < 256, big-endian 16-bit samples as uint16 otherwise"""
    with open(path, "rb") as f:
        data = f.read()
    tok, pos = [], 0
    while len(tok) < 4:
        while data[pos:pos + 1].isspace():
            pos += 1
        if data[pos:pos + 1] == b"#":
            pos = data.index(b"\n", pos) + 1; continue
        e = pos
        while not data[e:e + 1].isspace():
            e += 1
        tok.append(data[pos:e]); pos = e
    if tok[0] != b"P5":
        raise ValueError("not a binary PGM")
    w, h, mx = int(tok[1]), int(tok[2]), int(tok[3]); pos += 1
    dt = np.dtype(">u2") if mx > 255 else np.dtype(np.uint8)
    return np.frombuffer(data, dt, w * h, pos).reshape(h, w).astype(np.uint16 if mx > 255 else np.uint8)


def write_pgm(path: str, img):
    img = np.asarray(img)
    if img.dtype == np.uint16:
        body, mx = img.astype(">u2").tobytes(), 65535
    else:
        body, mx = np.asarray(img, np.uint8).tobytes(), 255
    with open(path, "wb") as f:
        f.write(b"P5\n%d %d\n%d\n" % (img.shape[1], img.shape[0], mx) + body)


class Undistort:
    """wOrg,hOrg: raw size; w,h: rectified size; K: 3x3 float64 (Undistort::getK()); remapX/remapY: (h,w) float32; passthrough: bool"""

    def __init__(self, parsOrg, wh_org, mode, wh):
        self.parsOrg = np.asarray(parsOrg, np.float64).copy()
        self.wOrg, self.hOrg = int(wh_org[0]), int(wh_org[1]); self.w, self.h = int(wh[0]), int(wh[1])
        self.passthrough = False; self.G = None; self.vignetteMapInv = None
        p = self.parsOrg
        if p[2] < 1 and p[3] < 1:                                              # "relative" calibration format (:736-755)
            p[0] = p[0] * self.wOrg; p[1] = p[1] * self.hOrg; p[2] = p[2] * self.wOrg - 0.5; p[3] = p[3] * self.hOrg - 0.5
        self.K = np.eye(3)
        if mode == "crop":
            self._make_optimal_K_crop()
        elif mode == "none":
            if (self.w, self.h) != (self.wOrg, self.hOrg):
                raise ValueError("rectification mode none requires input and output dimensions to match")
            self.K[0, 0], self.K[1, 1], self.K[0, 2], self.K[1, 2] = p[0], p[1], p[2], p[3]; self.passthrough = True
        elif mode == "full":
            raise NotImplementedError("makeOptimalK_full is `assert(false)` in the reference (Undistort.cpp:661-665)")
        else:                                                                  # explicit output calibration, relative to the image size (:824-837)
            oc = [f32(x) for x in mode]
            self.K[0, 0] = np.float64(oc[0] * f32(self.w)); self.K[1, 1] = np.float64(oc[1] * f32(self.h))
            self.K[0, 2] = np.float64(oc[2] * f32(self.w)) - 0.5; self.K[1, 2] = np.float64(oc[3] * f32(self.h)) - 0.5
        x, y = np.meshgrid(np.arange(self.w, dtype=f32), np.arange(self.h, dtype=f32))
        ix, iy = self._distort(x, y)
        ix = ix.copy(); iy = iy.copy()
        ix[ix == 0] = f32(0.001); iy[iy == 0] = f32(0.001)
        ix[ix == f32(self.wOrg - 1)] = f32(np.float64(self.wOrg) - 1.001)
        ix[iy == f32(self.hOrg - 1)] = f32(np.float64(self.hOrg) - 1.001)       # sic: the reference assigns ix here (:869)
        ok = (ix > 0) & (iy > 0) & (ix < f32(self.wOrg - 1)) & (iy < f32(self.wOrg - 1))   # sic: iy is tested against wOrg (:871)
        self.remapX = np.where(ok, ix, f32(-1)).astype(f32); self.remapY = np.where(ok, iy, f32(-1)).astype(f32)

    # UndistortPinhole::distortCoordinates (:1127-1152): float throughout, K read back as float
    def _distort(self, x, y):
        fx, fy, cx, cy = (_f32_of_f64(v) for v in self.parsOrg[:4])
        ofx, ofy, ocx, ocy = _f32_of_f64(self.K[0, 0]), _f32_of_f64(self.K[1, 1]), _f32_of_f64(self.K[0, 2]), _f32_of_f64(self.K[1, 2])
        x = np.asarray(x, f32); y = np.asarray(y, f32)
        ix = (x - ocx) / ofx; iy = (y - ocy) / ofy
        return fx * ix + cx, fy * iy + cy

    def _make_optimal_K_crop(self):
        w, h, wOrg, hOrg = self.w, self.h, self.wOrg, self.hOrg
        self.K = np.eye(3)
        t = (np.arange(100000, dtype=f32) - f32(50000.0)) / f32(10000.0); z = np.zeros(100000, f32)

        def span(vals, lim):                                                   # `if(minX==0) minX = t; maxX = t;` over the in-image samples
            idx = np.nonzero((vals > 0) & (vals < f32(lim)))[0]
            if len(idx) == 0:
                return f32(0), f32(0)
            nz = idx[t[idx] != 0]
            return (t[nz[0]] if len(nz) else f32(0)), t[idx[-1]]
        tx, _ = self._distort(t, z); minX, maxX = span(tx, wOrg - 1)
        _, ty = self._distort(z, t); minY, maxY = span(ty, hOrg - 1)
        minX, maxX, minY, maxY = (_f32_of_f64(np.float64(v) * 1.01) for v in (minX, maxX, minY, maxY))
        ys = np.arange(h, dtype=f32); xs = np.arange(w, dtype=f32)
        for iteration in range(1, 503):
            ry = minY + (maxY - minY) * ys / (f32(h) - f32(1.0))
            lx, _ = self._distort(np.full(h, minX, f32), ry); rx_, _ = self._distort(np.full(h, maxX, f32), ry)
            oobLeft = bool(np.any(~((lx > 0) & (lx < f32(wOrg - 1))))); oobRight = bool(np.any(~((rx_ > 0) & (rx_ < f32(wOrg - 1)))))
            rx = minX + (maxX - minX) * xs / (f32(w) - f32(1.0))
            _, ty_ = self._distort(rx, np.full(w, minY, f32)); _, by = self._distort(rx, np.full(w, maxY, f32))
            oobTop = bool(np.any(~((ty_ > 0) & (ty_ < f32(hOrg - 1))))); oobBottom = bool(np.any(~((by > 0) & (by < f32(hOrg - 1)))))
            if (oobLeft or oobRight) and (oobTop or oobBottom):
                if (maxX - minX) > (maxY - minY):
                    oobBottom = oobTop = False
                else:
                    oobLeft = oobRight = False
            if oobLeft: minX = _f32_of_f64(np.float64(minX) * 0.995)
            if oobRight: maxX = _f32_of_f64(np.float64(maxX) * 0.995)
            if oobTop: minY = _f32_of_f64(np.float64(minY) * 0.995)
            if oobBottom: maxY = _f32_of_f64(np.float64(maxY) * 0.995)
            if not (oobLeft or oobRight or oobTop or oobBottom):
                break
            if iteration > 500:
                raise RuntimeError("FAILED TO COMPUTE GOOD CAMERA MATRIX (Undistort.cpp:644-648)")
        k00 = (f32(w) - f32(1.0)) / (maxX - minX); k11 = (f32(h) - f32(1.0)) / (maxY - minY)
        self.K[0, 0] = np.float64(k00); self.K[1, 1] = np.float64(k11)
        self.K[0, 2] = np.float64(-minX) * self.K[0, 0]; self.K[1, 2] = np.float64(-minY) * self.K[1, 1]

    def set_photometric(self, pu: PhotometricUndistorter) -> "Undistort":
        """Undistort::loadPhotometricCalibration (:335-338): attach the PhotometricUndistorter of the raw size.  G / vignetteMapInv become what its
        processFrame applies at ingest (Context.setUndistort reads them), and photometricUndist.getG() is what src/main.cpp hands to setGammaFunction."""
        assert (pu.w, pu.h) == (self.wOrg, self.hOrg), "the photometric calibration has the raw image size"
        self.photometricUndist = pu; self.G = pu.ingest_G; self.vignetteMapInv = pu.ingest_vignetteMapInv
        return self

    @property
    def K4(self):
        """(fx, fy, cx, cy) as the float the pipeline keeps (setGlobalCalib(w, h, K.cast<float>()), src/main.cpp)"""
        return tuple(float(np.float32(v)) for v in (self.K[0, 0], self.K[1, 1], self.K[0, 2], self.K[1, 2]))

    @staticmethod
    def from_text(text: str) -> "Undistort":
        """Undistort::getUndistorterForFile (:232-334) for the Pinhole formats: "Pinhole fx fy cx cy 0" or a bare 5-number line ending in 0"""
        l = text.splitlines()
        if len(l) < 4:
            raise ValueError("calibration text needs 4 lines")
        tok = l[0].split()
        if tok and tok[0] == "Pinhole":
            tok = tok[1:]
        elif tok and tok[0] in ("FOV", "RadTan", "EquiDistant", "KannalaBrandt"):
            raise NotImplementedError(f"camera model {tok[0]}: only Pinhole is mirrored on the host (the device path takes any remap table)")
        pars = [float(v) for v in tok]
        if len(pars) != 5 or pars[4] != 0:
            raise NotImplementedError("only the distortion-free 5-parameter form is mirrored on the host")
        wh_org = [int(v) for v in l[1].split()[:2]]; wh = [int(v) for v in l[3].split()[:2]]
        mode = l[2].strip()
        if mode not in ("crop", "none", "full"):
            mode = [float(v) for v in mode.split()[:5]]
        return Undistort(pars, wh_org, mode, wh)

    @staticmethod
    def from_file(path: str) -> "Undistort":
        with open(path) as f:
            return Undistort.from_text(f.read())

    def undistort_host(self, raw_u8, factor=1.0):
        """numpy restatement of Undistort::undistort<unsigned char> without photometric calibration (test / data-preparation helper, float32 in the
        reference's operation order); the product path is the CUDA kernel."""
        raw = np.asarray(raw_u8); assert raw.shape == (self.hOrg, self.wOrg)
        src = (f32(factor) * raw.astype(f32)).reshape(-1)
        if self.passthrough:
            return src.reshape(self.h, self.w).copy()
        xx = self.remapX.reshape(-1); yy = self.remapY.reshape(-1); ok = xx >= 0
        xs = np.where(ok, xx, f32(1)); ysv = np.where(ok, yy, f32(1))
        xi = xs.astype(np.int32); yi = ysv.astype(np.int32)
        fx = xs - xi.astype(f32); fy = ysv - yi.astype(f32); xy = fx * fy
        o = xi + yi * self.wOrg
        out = xy * src[o + 1 + self.wOrg] + (fy - xy) * src[o + self.wOrg] + (fx - xy) * src[o + 1] + (f32(1) - fx - fy + xy) * src[o]
        return np.where(ok, out, f32(0)).astype(f32).reshape(self.h, self.w)
