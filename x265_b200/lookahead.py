"""Host mirror of the lookahead path (BASELINE configs[1] and [3]): Lowres::init (common/lowres.cpp:259-302) ->
LookaheadTLD::lowresIntraEstimate (encoder/slicetype.cpp:696-805) -> CostEstimateGroup::estimateFrameCost
(encoder/slicetype.cpp:3114-3214) on the device, through x265cu_frame_init_lowres / x265cu_lowres_intra_batch /
x265cu_lookahead_cost_batch (include/x265_b200.h).  Plumbing only: which (list, distance) motion fields exist, device
buffers, job records.  The arithmetic is all in libx265cu.so.

Frame sharding (SURVEY 8e, BASELINE configs[3]): every (p0, p1, b) estimate is independent of every other triple
(CostEstimateGroup batch mode, slicetype.cpp:1942-2009, 3027-3071), so frame b's estimates run on owner(b) = b % G.
The 4 half-pel planes of every frame are produced on its owner and published with ONE broadcast per frame
(`plane_block()` is the contiguous device range holding the 4 planes): the only data-path exchange.
"""
import numpy as np

MARGIN_X, MARGIN_Y = 96, 80               # Lowres / PicYuv luma margins (common/lowres.cpp:59-63, picyuv.cpp:87-88)
CMARGIN_X, CMARGIN_Y = 48, 40             # PicYuv 4:2:0 chroma margins
MVRANGE = 65536
LOOKAHEAD_LAMBDA = {8: 1.0, 10: 16.0}     # x265_lambda_tab[X265_LOOKAHEAD_QP = 12 + 6*(depth-8)] (constants.cpp:33-130)


def lowres_geometry(W, H):
    """(w8, h8, stride) of the lowres planes: widthInCU / heightInCU and the 32-aligned stride (lowres.cpp:51-63)."""
    w8 = ((W // 2) + 7) >> 3
    h8 = ((H // 2) + 7) >> 3
    stride = (W // 2 + 2 * MARGIN_X + 31) // 32 * 32
    return w8, h8, stride


def full_plane(img, depth):
    """Full-res luma in a PicYuv-like padded buffer (stride = CTU-aligned width + 2*96)."""
    H, W = img.shape
    dt = np.uint8 if depth == 8 else np.uint16
    stride = (W + 63) // 64 * 64 + 2 * MARGIN_X
    rows = (H + 63) // 64 * 64 + 2 * MARGIN_Y
    buf = np.zeros((rows, stride), dt)
    buf[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W] = img
    buf[MARGIN_Y:MARGIN_Y + H, :MARGIN_X] = img[:, :1]
    buf[MARGIN_Y:MARGIN_Y + H, MARGIN_X + W:MARGIN_X + W + MARGIN_X] = img[:, -1:]
    buf[:MARGIN_Y, :] = buf[MARGIN_Y:MARGIN_Y + 1, :]
    buf[MARGIN_Y + H:MARGIN_Y + H + MARGIN_Y, :] = buf[MARGIN_Y + H - 1:MARGIN_Y + H, :]
    return buf, stride, MARGIN_Y * stride + MARGIN_X


def coop_slices(H, lookahead_slices):
    """(numCoopSlices, numRowsPerSlice) as the Lookahead constructor settles them (slicetype.cpp:1016-1040): slices need a
    source height >= 720, at least 10 CU rows each; presets medium / slow ask for 8 / 4 (param.cpp:173, 492)."""
    h8 = ((H // 2) + 7) >> 3
    if lookahead_slices <= 1 or H < 720:
        return 1, h8
    rows = min(max(h8 // lookahead_slices, 10), h8)
    return h8 // rows, rows


def owner(poc, world):
    """Rank that owns lookahead frame `poc` (its lowres planes, intra costs and every estimate with b == poc)."""
    return poc % world


class _PlaneView:
    """A sub-range of a frame's plane block that quacks like a DeviceBuffer (ptr / nbytes / download)."""

    def __init__(self, block, offset, nbytes):
        self.block, self.offset, self.nbytes = block, offset, nbytes
        self.ptr = block.ptr + offset

    def download(self, dtype, count=None, offset=0):
        dt = np.dtype(dtype)
        if count is None:
            count = (self.nbytes - offset) // dt.itemsize
        return self.block.download(dtype, count, self.offset + offset)


class Lookahead:
    """Device-resident lookahead window of `nframes` frames of one geometry."""

    def __init__(self, lib, W, H, depth, nframes, lookahead_slices=0, keep_costs=False):
        """keep_costs: keep every estimate's per-CU lowresCosts resident on the device (Lowres::lowresCosts[b - p0][p1 - b]),
        as cu_tree() needs them; by default they live in a recycled per-launch block."""
        self.cu, self.depth, self.W, self.H, self.n = lib, depth, W, H, nframes
        self.keep_costs = keep_costs
        self.nslices, self.rows_per_slice = coop_slices(H, lookahead_slices)
        self.w8, self.h8, self.ls = lowres_geometry(W, H)
        self.ncu = self.w8 * self.h8
        self.es = 1 if depth == 8 else 2
        self.rows = self.h8 * 8 + 2 * MARGIN_Y
        self.plane_bytes = self.ls * self.rows * self.es
        self.lorg = (MARGIN_Y * self.ls + MARGIN_X) * self.es
        self.fr = []
        for _ in range(nframes):
            block = lib.alloc(4 * self.plane_bytes)            # the 4 hpel planes, contiguous: one broadcast per frame
            lib.check(lib.L.x265cu_memset(lib.ctx, block.ptr, 0, block.nbytes))
            planes = [_PlaneView(block, k * self.plane_bytes, self.plane_bytes) for k in range(4)]
            self.fr.append(dict(block=block, planes=planes, intraCost=lib.alloc(4 * self.ncu), intraMode=lib.alloc(self.ncu),
                                lc0=lib.alloc(2 * self.ncu), rs0=lib.alloc(4 * self.h8), out0=lib.alloc(16), mvs={}, mvcosts={}, res={}, lc={}, prop=None,
                                has_planes=False, has_intra=False, invq=None))
        self.tab = lib.to_device(lib.mvcost_table(LOOKAHEAD_LAMBDA[depth], MVRANGE))
        self._full = None
        self._chroma = None              # init_frame(aq=...): the staged 4:2:0 chroma pair
        self._pool = {}                  # size -> free device buffers: the per-step result / motion-field buffers are recycled
        lib.sync()                       # (a window's step made ~2000 cudaMalloc / cudaFree calls before: most of its host time)

    def _take(self, nbytes):
        free = self._pool.get(nbytes)
        return free.pop() if free else self.cu.alloc(nbytes)

    def _give(self, buf):
        self._pool.setdefault(buf.nbytes, []).append(buf)

    # ---- Lowres::init: full-res luma (host) -> 4 half-pel planes with extended borders (device) ----
    def init_frame(self, i, img, sync=True, *, cb=None, cr=None, aq=None, keep_chroma=False):
        """Lowres::init of frame i from its full-resolution luma (host array, ideally pinned): strided H2D straight into the
        PicYuv-like padded device plane, border extension (pixel.cpp:1027-1041) and the lowres kernel on the device.

        aq: None (the frame's invQscale comes from set_invqscale, if at all), or a dict of calcAdaptiveQuantFrame's
        parameters: mode (rc.aqMode 0-3), strength, qg_size, weightp, variance, quant_offsets (blockCount floats or None).
        Then the 4:2:0 chroma planes cb / cr (host, W / 2 x H / 2; None for 4:0:0) are staged next to the luma, the AQ pass
        runs on the device and its host finish leaves the frame's invQscale resident (invQscaleFactor8x8 at qg_size 8), and
        the frame record keeps qpAqOffset, wp_sum and wp_ssd (and blockVariance / frameVariance with variance).

        keep_chroma: keep cb / cr resident for this frame in PicYuv-like buffers (48 x 40 margins, borders extended), as
        weight_analyse() reads them."""
        cu = self.cu
        img = np.ascontiguousarray(img)
        H, W = img.shape
        fs = (W + 63) // 64 * 64 + 2 * MARGIN_X
        rows = (H + 63) // 64 * 64 + 2 * MARGIN_Y
        forg = (MARGIN_Y * fs + MARGIN_X) * self.es
        if self._full is None:
            self._full = cu.alloc(fs * rows * self.es)
            cu.check(cu.L.x265cu_memset(cu.ctx, self._full.ptr, 0, self._full.nbytes))
        cu.check(cu.L.x265cu_copy2d(cu.ctx, self._full.ptr + forg, fs * self.es, img.ctypes.data, W * self.es, W * self.es, H, 0))
        cu.check(cu.L.x265cu_extend_border(cu.ctx, self.depth, self._full.ptr + forg, fs, W, H, MARGIN_X, MARGIN_Y))
        f = self.fr[i]
        cu.check(cu.L.x265cu_frame_init_lowres(cu.ctx, self.depth, self._full.ptr + forg, fs,
                                               *[p.ptr + self.lorg for p in f["planes"]], self.ls, self.w8 * 8, self.h8 * 8, MARGIN_X, MARGIN_Y))
        if aq is not None:
            self._aq_frame(i, self._full.ptr + forg, fs, W, H, cb, cr, aq)
        # weight_analyse reads only what this init_frame left: the statistics of its AQ pass and the chroma it kept
        self.fr[i]["wp_valid"] = aq is not None
        if keep_chroma:
            self._keep_chroma(i, cb, cr)
        else:
            for buf in self.fr[i].pop("chroma", None) or []:      # a re-used slot must not keep the previous frame's chroma
                buf.free()
        if sync:
            cu.sync()          # the host image may be released / the staging plane re-used
        f["has_planes"] = True

    def _aq_frame(self, i, luma, fs, W, H, cb, cr, aq):
        """calcAdaptiveQuantFrame of frame i through x265cu_aq_frame, on the staged planes."""
        import ctypes as C
        from .lib import AqParams, AqOut, aq_geometry
        cu = self.cu
        assert (cb is None) == (cr is None), "give both chroma planes or neither"
        cw, chh = W // 2, H // 2
        cptr = [None, None]
        if cb is not None:
            if self._chroma is None:
                self._chroma = [cu.alloc(cw * chh * self.es) for _ in range(2)]
            for k, pl in enumerate((cb, cr)):
                pl = np.ascontiguousarray(pl)
                assert pl.shape == (chh, cw)
                cu.check(cu.L.x265cu_copy2d(cu.ctx, self._chroma[k].ptr, cw * self.es, pl.ctypes.data, cw * self.es, cw * self.es, chh, 0))
                cptr[k] = self._chroma[k].ptr
        qg = int(aq.get("qg_size", 32))
        _, count, _ = aq_geometry(W, H, qg)
        qo = aq.get("quant_offsets")
        qo = None if qo is None else np.ascontiguousarray(qo, np.float32)
        assert qo is None or qo.size == count
        prm = AqParams(aqMode=int(aq.get("mode", 2)), qgSize=qg, weightp=int(bool(aq.get("weightp", False))),
                       variance=int(bool(aq.get("variance", False))), aqStrength=float(aq.get("strength", 1.0)),
                       quantOffsets=qo.ctypes.data if qo is not None else None)
        f = self.fr[i]
        rec = dict(qpAqOffset=np.zeros(count), wp_sum=np.zeros(3, np.uint64), wp_ssd=np.zeros(3, np.uint64))
        if prm.variance:
            rec.update(blockVariance=np.zeros(count, np.uint32), frameVariance=np.zeros(1))
        out = AqOut(**{k: v.ctypes.data for k, v in rec.items()})
        if prm.aqMode != 0 and f["invq"] is None:
            f["invq"] = cu.alloc(4 * self.ncu)
        cu.check(cu.L.x265cu_aq_frame(cu.ctx, self.depth, luma, fs, cptr[0], cptr[1], cw, W, H, C.byref(prm),
                                      f["invq"].ptr if prm.aqMode != 0 else None, C.byref(out)))
        if prm.variance:
            rec["frameVariance"] = float(rec["frameVariance"][0])
        f.update(rec)

    def _keep_chroma(self, i, cb, cr):
        """frame i's 4:2:0 chroma in its own padded buffers, borders extended (the reference's m_bChromaExtended)"""
        cu = self.cu
        cw, chh = self.W // 2, self.H // 2
        cs = ((self.W + 63) // 64 * 64) // 2 + 2 * CMARGIN_X
        rows = ((self.H + 63) // 64 * 64) // 2 + 2 * CMARGIN_Y
        corg = (CMARGIN_Y * cs + CMARGIN_X) * self.es
        f = self.fr[i]
        if f.get("chroma") is None:
            f["chroma"] = [cu.alloc(cs * rows * self.es) for _ in range(2)]
        for buf, pl in zip(f["chroma"], (cb, cr)):
            pl = np.ascontiguousarray(pl)
            assert pl.shape == (chh, cw)
            cu.check(cu.L.x265cu_copy2d(cu.ctx, buf.ptr + corg, cs * self.es, pl.ctypes.data, cw * self.es, cw * self.es, chh, 0))
            cu.check(cu.L.x265cu_extend_border(cu.ctx, self.depth, buf.ptr + corg, cs, cw, chh, CMARGIN_X, CMARGIN_Y))
        f["cstride"], f["corg"] = cs, corg

    def _wp_frame(self, i):
        from .lib import WpFrame
        f = self.fr[i]
        if not f.get("wp_valid"):
            raise ValueError("frame %d has no picture statistics: init_frame it with aq={...}" % i)
        r = WpFrame()
        for k in range(4):
            r.lowres[k] = f["planes"][k].ptr + self.lorg
        r.lowresStride = self.ls
        if f.get("chroma") is not None:
            r.cb, r.cr = f["chroma"][0].ptr + f["corg"], f["chroma"][1].ptr + f["corg"]
            r.chromaStride = f["cstride"]
        for k in range(3):
            r.wp_sum[k], r.wp_ssd[k] = int(f["wp_sum"][k]), int(f["wp_ssd"][k])
        r.poc = i
        return r

    def weight_analyse(self, b, slice_type, refs, bframes, num_ref_idx):
        """weightAnalyse (encoder/weightPrediction.cpp:222-539) of frame b as a P (slice_type "P", refs = [ref0]) or B
        ("B", refs = [ref0, ref1]) slice, on what the window holds: the lowres planes, intraCost, the motion fields
        lowresMvs[list][|b - ref|] (those the estimates searched), wp_sum / wp_ssd (init_frame(aq=...)) and, in 4:2:0,
        the chroma kept by init_frame(keep_chroma=True) (4:0:0 when frame b has none).  Window indices are the pocs.
        num_ref_idx: Slice::m_numRefIdx per list.  Returns the [2][16][3][4] int32 table of {wtPresent, inputWeight,
        log2WeightDenom, inputOffset}; entries the reference does not write stay 0."""
        import ctypes as C
        from .lib import WpParams, WpFrame
        cu = self.cu
        nl = 1 if slice_type == "P" else 2
        assert len(refs) == nl and self.fr[b]["has_intra"]
        csp = 1 if self.fr[b].get("chroma") is not None else 0
        prm = WpParams(1 if nl == 1 else 0, (C.c_int32 * 2)(*(list(num_ref_idx) + [0] * (2 - len(num_ref_idx)))), bframes,
                       self.W, self.H, csp)
        fenc = self._wp_frame(b)
        recs = [self._wp_frame(r) for r in refs]
        rp = (C.POINTER(WpFrame) * 2)(*[C.pointer(r) for r in recs] + [C.POINTER(WpFrame)()] * (2 - nl))
        mvs = (C.c_void_p * 2)()
        for lst, r in enumerate(refs):
            mv = self.fr[b]["mvs"].get((lst, abs(b - r)))
            mvs[lst] = mv.ptr if mv is not None else None
        out = np.zeros((2, 16, 3, 4), np.int32)
        cu.check(cu.L.x265cu_weightp_analyse(cu.ctx, self.depth, C.byref(prm), C.byref(fenc), self.fr[b]["intraCost"].ptr, rp,
                                             mvs, out.ctypes.data))
        return out

    def set_invqscale(self, i, invq):
        """Lowres::invQscaleFactor of frame i (int32 per lowres CU, 256 = 1.0): the adaptive-quantisation weights that
        calcAdaptiveQuantFrame (slicetype.cpp:444-694, host float math) produced; costEstAq and the row sums use them."""
        a = np.ascontiguousarray(invq, np.int32)
        assert a.size == self.ncu
        f = self.fr[i]
        if f["invq"] is None:
            f["invq"] = self.cu.alloc(4 * self.ncu)
        f["invq"].upload(a)

    def plane_block(self, i):
        """(device pointer, bytes) of frame i's 4 planes: what its owner broadcasts."""
        b = self.fr[i]["block"]
        return b.ptr, b.nbytes

    def planes_received(self, i):
        self.fr[i]["has_planes"] = True

    # ---- lowresIntraEstimate for a set of frames: one launch ----
    def intra_batch(self, ids):
        from .lib import LA_INTRA_JOB
        cu = self.cu
        ids = [i for i in ids if not self.fr[i]["has_intra"]]
        if not ids:
            return
        jobs = np.zeros(len(ids), LA_INTRA_JOB)
        for n, i in enumerate(ids):
            f = self.fr[i]
            assert f["has_planes"], "frame %d has no lowres planes on this rank" % i
            j = jobs[n]
            j["plane0"] = f["planes"][0].ptr + self.lorg; j["invQscale"] = f["invq"].ptr if f["invq"] is not None else 0; j["intraCost"] = f["intraCost"].ptr; j["intraMode"] = f["intraMode"].ptr
            j["lowresCosts"] = f["lc0"].ptr; j["rowSatds"] = f["rs0"].ptr; j["out"] = f["out0"].ptr
        d_jobs = cu.to_device(jobs)
        cu.check(cu.L.x265cu_lowres_intra_batch(cu.ctx, self.depth, d_jobs.ptr, len(ids), self.ls, self.w8, self.h8, int(LOOKAHEAD_LAMBDA[self.depth])))
        cu.sync()
        d_jobs.free()
        for i in ids:
            self.fr[i]["has_intra"] = True

    def cost(self, p0, p1, b):
        return self.cost_batch([(p0, p1, b)])[0]

    def prepare_batch(self, triples):
        """Job records of the not-yet-estimated triples (uploaded), result buffers allocated: the launch itself is
        launch_batch().  The triples of one batch must not share a motion field that still has to be searched."""
        from .lib import LA_JOB
        cu = self.cu
        todo = [t for t in triples if (t[2] - t[0], t[1] - t[2]) not in self.fr[t[2]]["res"]]
        recs = []
        bufs = []
        # the batch's results land in three blocks (per-CU costs, row sums, frame totals): one D2H each in collect_batch()
        nt = len(todo)
        lcB = self._take(2 * self.ncu * nt) if nt and not self.keep_costs else None
        rsB = self._take(4 * self.h8 * nt) if nt else None
        outB = self._take(32 * nt) if nt else None
        for ti, (p0, p1, b) in enumerate(todo):
            f = self.fr[b]
            assert f["has_intra"] and self.fr[p0]["has_planes"] and self.fr[p1]["has_planes"], (p0, p1, b)
            d0, d1 = b - p0, p1 - b
            j = np.zeros(1, LA_JOB)[0]
            for k in range(4):
                j["fenc"][k] = f["planes"][k].ptr + self.lorg
                j["ref0"][k] = self.fr[p0]["planes"][k].ptr + self.lorg
                j["ref1"][k] = self.fr[p1]["planes"][k].ptr + self.lorg
            j["bidir"] = int(b < p1)
            for lst, dist in ((0, d0), (1, d1)):
                new = (lst, dist) not in f["mvs"]
                if new:
                    f["mvs"][(lst, dist)] = self._take(8 * self.ncu); f["mvcosts"][(lst, dist)] = self._take(4 * self.ncu)
                    cu.check(cu.L.x265cu_memset(cu.ctx, f["mvs"][(lst, dist)].ptr, 0, 8 * self.ncu))
                    cu.check(cu.L.x265cu_memset(cu.ctx, f["mvcosts"][(lst, dist)].ptr, 0, 4 * self.ncu))
                j["doSearch%d" % lst] = int(new and (lst == 0 or p1 > b))
                j["mvs"][lst] = f["mvs"][(lst, dist)].ptr; j["mvcosts"][lst] = f["mvcosts"][(lst, dist)].ptr
            if self.keep_costs:
                lc = f["lc"][(d0, d1)] = self._take(2 * self.ncu)
            else:
                lc = _PlaneView(lcB, ti * 2 * self.ncu, 2 * self.ncu)
            rs = _PlaneView(rsB, ti * 4 * self.h8, 4 * self.h8); out = _PlaneView(outB, ti * 32, 24)
            bufs.append((lc, rs, out))
            j["intraCost"] = f["intraCost"].ptr; j["invQscale"] = f["invq"].ptr if f["invq"] is not None else 0; j["lowresCosts"] = lc.ptr; j["rowSatds"] = rs.ptr; j["out"] = out.ptr
            # cooperative slices (slicetype.cpp:3143): one job per slice, each an independent wavefront over its CU rows
            if self.nslices > 1 and (p1 > b or j["doSearch0"] or j["doSearch1"]):
                for sl in range(self.nslices):
                    y0 = self.rows_per_slice * sl
                    y1 = self.h8 if sl == self.nslices - 1 else self.rows_per_slice * (sl + 1)
                    js = j.copy(); js["rows"] = y0 | (y1 << 16)
                    recs.append(js)
            else:
                recs.append(j)
        jobs = np.array(recs, LA_JOB) if recs else np.zeros(1, LA_JOB)
        d_j = None
        if todo:
            d_j = self._take((jobs.nbytes + 65535) // 65536 * 65536)
            d_j.upload(jobs)
        return dict(todo=todo, bufs=bufs, d_jobs=d_j, njobs=len(recs), blocks=(lcB, rsB, outB))

    def launch_batch(self, prep):
        """ONE kernel launch for all prepared triples (asynchronous on the context's stream)."""
        cu = self.cu
        if prep["todo"]:
            cu.check(cu.L.x265cu_lookahead_cost_batch(cu.ctx, self.depth, prep["d_jobs"].ptr, prep["njobs"], self.ls, self.w8, self.h8,
                                                      self.tab.ptr + 2 * MVRANGE))

    def collect_batch(self, prep, full=True):
        """D2H of the launched triples' results: frame cost always; per-CU lowresCosts / rowSatds when `full`."""
        lcB, rsB, outB = prep["blocks"]
        nt = len(prep["todo"])
        if nt:
            outs = outB.download(np.int64, 4 * nt).reshape(nt, 4)
            lcs = None
            if full:
                lcs = np.stack([lc.download(np.uint16, self.ncu) for lc, _, _ in prep["bufs"]]) if self.keep_costs else \
                    lcB.download(np.uint16, self.ncu * nt).reshape(nt, self.ncu)
            rss = rsB.download(np.int32, self.h8 * nt).reshape(nt, self.h8) if full else None
        for ti, (p0, p1, b) in enumerate(prep["todo"]):
            o = outs[ti]
            score = int(o[0])
            if b != p1:
                score = score * 100 // 130          # slicetype.cpp:3205-3206, bFrameBias = 0
            r = dict(score=score, costEstAq=int(o[1]), intraMbs=int(o[2]))
            if full:
                r["lowresCosts"] = lcs[ti].copy(); r["rowSatds"] = rss[ti].copy()
            self.fr[b]["res"][(b - p0, p1 - b)] = r
        for blk in (lcB, rsB, outB, prep["d_jobs"]):
            if blk is not None:
                self._give(blk)

    def cost_batch(self, triples, full=True):
        """Frame costs of `triples` (one launch for those not estimated yet)."""
        prep = self.prepare_batch(triples)
        self.launch_batch(prep)
        self.collect_batch(prep, full)
        return [self.fr[b]["res"][(b - p0, p1 - b)]["score"] for (p0, p1, b) in triples]

    def forget_results(self):
        """Drop cached estimates and motion fields (bench: re-run the same window)."""
        for f in self.fr:
            for d in (f["mvs"], f["mvcosts"], f["lc"]):
                for v in d.values():
                    self._give(v)
                d.clear()
            f["res"].clear()

    def close(self):
        self.forget_results()
        for f in self.fr:
            for k in ("block", "intraCost", "intraMode", "lc0", "rs0", "out0"):
                f[k].free()
            if f["invq"] is not None:
                f["invq"].free()
            if f["prop"] is not None:
                f["prop"].free()
            for buf in f.get("chroma") or []:
                buf.free()
        self.tab.free()
        if self._full is not None:
            self._full.free()
        for b in self._chroma or []:
            b.free()
        self._chroma = None
        for free in self._pool.values():
            for b in free:
                b.free()
        self._pool.clear()


    # ---- cuTree: Lookahead::cuTree's propagation chain on the device (x265cu_cutree) ----
    def cu_tree(self, slice_types, b_intra=False, lookahead_depth=40, b_pyramid=True, weighted_bipred=False, vbv=False, fps=(25, 1),
                world=1, rank=0):
        """Lookahead::cuTree (slicetype.cpp:2538-2639) over frames 0..len(slice_types)-1 of the window, up to cuTreeFinish.
        Computes the estimates the chain reads that are not resident yet (cost_batch, in conflict-free launches), runs the
        chain on the device and downloads only the propagateCost of the frames cuTreeFinish is then called on.
        Returns (finish, costs): finish = [(frame, ref0Distance)] in the reference's order (-1: the lookahead-less intra case,
        qpAqOffset copied), costs = {frame: propagateCost (uint16 per lowres CU)}.  Needs keep_costs=True and every frame's
        invQscale (set_invqscale: invQscaleFactor, or invQscaleFactor8x8 when rc.qgSize == 8).  With frame shards
        (world > 1) every estimate must live on this rank: cuTree across ranks is not supported."""
        from .lib import CutreeFrame, CutreeParams
        import ctypes as C
        cu = self.cu
        if not self.keep_costs:
            raise ValueError("cu_tree needs the estimates' lowresCosts resident: construct Lookahead with keep_costs=True")
        numframes = len(slice_types) - 1
        if numframes < 0 or numframes >= self.n:
            raise ValueError("cu_tree: %d frames, the window holds %d" % (numframes + 1, self.n))
        prm = CutreeParams(int(b_intra), lookahead_depth, int(b_pyramid), int(weighted_bipred), int(vbv), fps[0], fps[1])
        st = np.ascontiguousarray(slice_types, np.int32)
        cap = 4 * (numframes + 2) * 18
        tri = np.zeros(3 * cap, np.int32)
        n = cu.L.x265cu_cutree_estimates(st.ctypes.data, numframes, C.byref(prm), tri.ctypes.data, cap)
        if n < 0:
            raise RuntimeError(cu.last_error())
        triples = [tuple(int(v) for v in tri[3 * k:3 * k + 3]) for k in range(n)]
        for (p0, p1, b) in triples:
            if owner(b, world) != rank:
                raise ValueError("cu_tree: estimate (%d, %d, %d) lives on rank %d, not on rank %d; cuTree across lookahead frame "
                                 "shards is not supported" % (p0, p1, b, owner(b, world), rank))
        missing = [t for t in dict.fromkeys(triples) if (t[2] - t[0], t[1] - t[2]) not in self.fr[t[2]]["res"]]
        for batch in conflict_free_batches(missing):
            self.cost_batch(batch, full=False)
        recs = (CutreeFrame * (numframes + 1))()
        byptr = {}
        for i in range(numframes + 1):
            f = self.fr[i]
            if f["prop"] is None:
                f["prop"] = cu.alloc(2 * self.ncu)
            byptr[f["prop"].ptr] = f["prop"]
            r = recs[i]
            r.intraCost = f["intraCost"].ptr
            r.invQscale = f["invq"].ptr if f["invq"] is not None else None
            r.propagateCost = f["prop"].ptr
            r.sliceType = int(st[i])
            for (d0, d1), lc in f["lc"].items():
                r.lowresCosts[d0][d1] = lc.ptr
            for (lst, dist), mv in f["mvs"].items():
                r.mvs[lst][dist] = mv.ptr
        fin = np.zeros(2 * (numframes + 2), np.int32)
        nf = cu.L.x265cu_cutree(cu.ctx, recs, numframes, C.byref(prm), self.w8, self.h8, fin.ctypes.data, numframes + 2)
        if nf < 0:
            raise RuntimeError(cu.last_error())
        for i in range(numframes + 1):                 # the reference's propagateCost pointer swaps
            self.fr[i]["prop"] = byptr[recs[i].propagateCost]
        finish = [(int(fin[2 * k]), int(fin[2 * k + 1])) for k in range(nf)]
        costs = {f: self.fr[f]["prop"].download(np.uint16, self.ncu) for f, d in finish if d >= 0}
        return finish, costs


def window_triples(nframes, bframes):
    """The (p0, p1, b) estimates slicetypeDecide's cost passes issue for a window with `bframes` B-frames between anchors
    (slicetype.cpp:1942-2009: P costs of every anchor distance and the B costs between them): the bench / shard workload."""
    out = []
    for b in range(1, nframes):
        for d in range(1, min(bframes + 1, b) + 1):
            out.append((b - d, b, b))                     # P estimate at distance d
    for p0 in range(0, nframes - 2):
        for p1 in range(p0 + 2, min(p0 + bframes + 1, nframes - 1) + 1):
            for b in range(p0 + 1, p1):
                out.append((p0, p1, b))                   # B estimate inside (p0, p1)
    return out


def conflict_free_batches(triples):
    """Split triples into launches such that no two triples of a launch search the same motion field
    (frame b, list, distance): x265cu_lookahead_cost_batch runs its triples concurrently."""
    batches = []
    for t in triples:
        p0, p1, b = t
        keys = {(b, 0, b - p0)} | ({(b, 1, p1 - b)} if p1 > b else set())
        for bt in batches:
            if not (bt["keys"] & keys):
                bt["t"].append(t); bt["keys"] |= keys
                break
        else:
            batches.append(dict(t=[t], keys=set(keys)))
    return [bt["t"] for bt in batches]
