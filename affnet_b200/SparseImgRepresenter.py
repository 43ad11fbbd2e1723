"""ScaleSpaceAffinePatchExtractor with the reference's interface (SparseImgRepresenter.py:14-209), executed by
the sm_90a CUDA library: Gaussian pyramid -> fused Hessian/NMS/soft-argmax detection -> device-side selection ->
affine patch sampling -> AffNet -> shape filter -> (OriNet) -> denormalised LAFs.

Differences from the reference that a caller can observe: nothing is printed; inputs must be CUDA tensors (there
is no CPU path); `pyr_idxs` / `level_idxs` may be given as float or int tensors (returned as float, as the
reference does).  AffNet=None / OriNet=None select the hand-crafted estimators (Baumberg step, gradient-histogram
orientation) exactly as the reference does; a custom RespNet is not supported.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib as L
from .HandCraftedModules import AffineShapeEstimator, OrientationDetector, ScalePyramid
from .LAF import denormalizeLAFs, get_pyramid_and_level_index_for_LAFs, normalizeLAFs


def angles2A(angles):
    """LAF.py:306-311."""
    c, s = torch.cos(angles).view(-1, 1, 1), torch.sin(angles).view(-1, 1, 1)
    return torch.cat([torch.cat([c, s], dim=2), torch.cat([-s, c], dim=2)], dim=1)


class ScaleSpaceAffinePatchExtractor(nn.Module):
    def __init__(self, border=16, num_features=500, patch_size=32, mrSize=3.0, nlevels=3, num_Baum_iters=0,
                 init_sigma=1.6, th=None, RespNet=None, OriNet=None, AffNet=None):
        super().__init__()
        self.mrSize = mrSize
        self.PS = patch_size
        self.b = border
        self.num = num_features
        self.nlevels = nlevels
        self.num_Baum_iters = num_Baum_iters
        self.init_sigma = init_sigma
        self.th = th
        if th is not None:          # SparseImgRepresenter.py:33-37
            self.num = -1
        else:
            self.th = 0
        if RespNet is not None:
            raise NotImplementedError("custom RespNet: only the fused Hessian response is implemented")
        # SparseImgRepresenter.py:42-49: the hand-crafted estimators are the defaults
        self.OriNet = OriNet if OriNet is not None else OrientationDetector(patch_size=19)
        self.AffNet = AffNet if AffNet is not None else AffineShapeEstimator(patch_size=19)
        self.ScalePyrGen = ScalePyramid(nLevels=nlevels, init_sigma=init_sigma, border=border)
        self._plan = None
        self._pyr_buf = None
        self.scale_pyr, self.sigmas, self.pix_dists = None, None, None

    # ---- detection -----------------------------------------------------------------------------------------
    def _build_pyramid(self, x):
        x = L.f32c(x, "x")
        if x.dim() != 4 or x.size(0) != 1 or x.size(1) != 1:
            raise L.AffnetB200Error("expected an image of shape [1,1,H,W]")
        self._plan, self._pyr_buf = self.ScalePyrGen.build(x)
        self.scale_pyr, self.sigmas, self.pix_dists = ScalePyramid.views(self._plan, self._pyr_buf)
        return x

    def _detect(self, num_features, a_scale):
        plan, dev = self._plan, self._pyr_buf.device
        lib = L.lib()
        cap = max(plan.H * plan.W // 16, 4096, num_features)
        while True:
            nbytes = lib.ag_detect_ws_bytes(C.byref(plan), cap)
            ws_buf = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            ws = L.DetectWs()
            L.check(lib.ag_detect_ws_carve(C.byref(plan), cap, L.ptr(ws_buf), C.byref(ws)))
            L.check(lib.ag_detect(C.byref(plan), L.ptr(self._pyr_buf), float(self.th), int(self.mrSize), C.byref(ws), L.stream_ptr()))
            if num_features > 0:
                out_cap = num_features
                resp, lafs, oct_, lvl, cnt = self._select_outputs(out_cap, dev)
                # any count: the shared-memory sort up to 16384 keypoints, the global-memory one above (no scratch below)
                scratch = self._scratch(lib.ag_select_topk_workspace_bytes(C.byref(plan), cap, out_cap), dev)
                L.check(lib.ag_select_topk_keypoints(C.byref(plan), C.byref(ws), num_features, float(a_scale), out_cap, L.ptr(scratch),
                                                     0 if scratch is None else scratch.numel(), L.ptr(resp), L.ptr(lafs), L.ptr(oct_),
                                                     L.ptr(lvl), L.ptr(cnt), L.stream_ptr()))
                # one host round trip: candidate count (overflow check) + selected count
                host = torch.cat([self._wrap_i32(ws.d_cand_count, 1, ws_buf), cnt]).cpu()
            else:
                host = self._wrap_i32(ws.d_cand_count, 1, ws_buf).cpu()
            n_cand = int(host[0])
            if n_cand > cap:
                cap = n_cand + 1024
                continue
            if num_features <= 0:
                # th mode: every candidate of the accepted levels in (octave, level, raster) order; the candidate count bounds them
                resp, lafs, oct_, lvl, cnt = self._select_outputs(max(n_cand, 1), dev)
                scratch = torch.empty(lib.ag_select_all_workspace_bytes(C.byref(plan), cap), dtype=torch.uint8, device=dev)
                L.check(lib.ag_select_all_keypoints(C.byref(plan), C.byref(ws), float(a_scale), max(n_cand, 1), L.ptr(scratch),
                                                    scratch.numel(), L.ptr(resp), L.ptr(lafs), L.ptr(oct_), L.ptr(lvl), L.ptr(cnt),
                                                    L.stream_ptr()))
                host = cnt.cpu()
            n = int(host[-1])
            return resp[:n], lafs[:n], oct_[:n], lvl[:n]

    @staticmethod
    def _select_outputs(n, dev):
        return (torch.empty(n, dtype=torch.float32, device=dev), torch.empty(n, 2, 3, dtype=torch.float32, device=dev),
                torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
                torch.empty(1, dtype=torch.int32, device=dev))

    @staticmethod
    def _scratch(nbytes, dev):
        """Scratch of a top-K entry point, or None when it needs none."""
        return torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None

    @staticmethod
    def _wrap_i32(addr, n, owner):
        """View `n` int32 at device address `addr` inside `owner` (a uint8 tensor)."""
        off = addr - owner.data_ptr()
        return owner[off:off + 4 * n].view(torch.int32)

    def multiScaleDetector(self, x, num_features=0):
        """SparseImgRepresenter.py:53-111 -> (responses, LAFs normalised (A not yet scaled by mrSize), pyr_idxs, level_idxs)."""
        self._build_pyramid(x)
        resp, lafs, oct_, lvl = self._detect(num_features, 1.0)
        return resp, lafs, oct_.float(), lvl.float()

    # ---- patches from the cached pyramid ---------------------------------------------------------------------
    def _patches(self, LAFs, oct_, lvl, PS):
        n = LAFs.size(0)
        out = torch.empty(n, 1, PS, PS, dtype=torch.float32, device=LAFs.device)
        LAFs = L.f32c(LAFs)
        oct_ = oct_.to(torch.int32).contiguous()
        lvl = lvl.to(torch.int32).contiguous()
        step = 65535
        for s in range(0, n, step):
            e = min(n, s + step)
            L.check(L.lib().ag_extract_patches_pyr(C.byref(self._plan), L.ptr(self._pyr_buf), L.ptr(LAFs[s:e]), L.ptr(oct_[s:e]),
                                                   L.ptr(lvl[s:e]), None, e - s, PS, L.ptr(out[s:e]), L.stream_ptr()))
        return out

    # ---- affine shape -------------------------------------------------------------------------------------------
    def getAffineShape(self, final_resp, LAFs, final_pyr_idxs, final_level_idxs, num_features=0):
        """SparseImgRepresenter.py:113-165."""
        n = LAFs.size(0)
        dev = LAFs.device
        LAFs = L.f32c(LAFs)
        final_resp = L.f32c(final_resp)
        oct_ = final_pyr_idxs.to(torch.int32).contiguous()
        lvl = final_level_idxs.to(torch.int32).contiguous()
        base_A = None
        cur = LAFs
        lib = L.lib()
        for i in range(self.num_Baum_iters):
            patches = self._patches(cur, oct_, lvl, self.AffNet.PS)
            A = L.f32c(self.AffNet(patches))
            if base_A is None:
                base_A = A
            elif n:
                nb = torch.empty_like(A)
                L.check(lib.ag_mat2_compose(L.ptr(A), L.ptr(L.f32c(base_A)), L.ptr(nb), n, L.stream_ptr()))      # base_A <- A base_A (:133)
                base_A = nb
            if i != self.num_Baum_iters - 1 and n:
                cur = torch.empty_like(LAFs)
                L.check(lib.ag_lafs_left_multiply(L.ptr(L.f32c(base_A)), L.ptr(LAFs), L.ptr(cur), n, L.stream_ptr()))   # (:134-135)
        if base_A is None:
            base_A = torch.eye(2, device=dev).unsqueeze(0).expand(n, 2, 2)
        base_A = L.f32c(base_A)
        resp_o = torch.empty(n, dtype=torch.float32, device=dev)
        lafs_o = torch.empty(n, 2, 3, dtype=torch.float32, device=dev)
        oct_o = torch.empty(n, dtype=torch.int32, device=dev)
        lvl_o = torch.empty(n, dtype=torch.int32, device=dev)
        cnt_in = torch.tensor([n], dtype=torch.int32, device=dev)
        cnt_o = torch.empty(1, dtype=torch.int32, device=dev)
        if n > 0 and num_features <= 0:
            # every survivor in order (:151-156), at any n
            L.check(L.lib().ag_affine_shape_filter_all(L.ptr(base_A), L.ptr(final_resp), L.ptr(LAFs), L.ptr(oct_), L.ptr(lvl), L.ptr(cnt_in),
                                                       1, n, L.ptr(resp_o), L.ptr(lafs_o), L.ptr(oct_o), L.ptr(lvl_o), L.ptr(cnt_o),
                                                       L.stream_ptr()))
            m = int(cnt_o.item())
        elif n > 0:
            scratch = self._scratch(lib.ag_affine_shape_filter_topk_workspace_bytes(1, n), dev)
            L.check(lib.ag_affine_shape_filter_topk(L.ptr(base_A), L.ptr(final_resp), L.ptr(LAFs), L.ptr(oct_), L.ptr(lvl), L.ptr(cnt_in),
                                                    1, n, int(num_features), n, L.ptr(scratch), 0 if scratch is None else scratch.numel(),
                                                    L.ptr(resp_o), L.ptr(lafs_o), L.ptr(oct_o), L.ptr(lvl_o), L.ptr(cnt_o), L.stream_ptr()))
            m = int(cnt_o.item())
        else:
            m = 0
        return resp_o[:m], lafs_o[:m], oct_o[:m].float(), lvl_o[:m].float()

    # ---- orientation --------------------------------------------------------------------------------------------
    def getOrientation(self, LAFs, final_pyr_idxs, final_level_idxs):
        """SparseImgRepresenter.py:167-180 (without the reference's discarded second extraction)."""
        patches = self._patches(LAFs, final_pyr_idxs, final_level_idxs, self.OriNet.PS)
        angles = self.OriNet(patches)
        R = angles if angles.dim() > 2 else angles2A(angles).view(-1, 2, 2)
        out = L.f32c(LAFs).clone()
        if out.size(0):
            L.check(L.lib().ag_lafs_apply_rotation(L.ptr(out), L.ptr(L.f32c(R)), out.size(0), L.stream_ptr()))
        return out

    def extract_patches_from_pyr(self, dLAFs, PS=41):
        """SparseImgRepresenter.py:181-188."""
        if self._plan is None:
            raise L.AffnetB200Error("extract_patches_from_pyr needs a prior forward() (it samples the cached pyramid)")
        o, l = get_pyramid_and_level_index_for_LAFs(dLAFs, self._plan, PS)
        return self._patches(normalizeLAFs(dLAFs, self._plan.W, self._plan.H), o, l, PS)

    def forward(self, x, do_ori=False):
        """SparseImgRepresenter.py:189-209 -> (dLAFs [N,2,3] in pixels, responses [N])."""
        x = self._build_pyramid(x)
        nf = self.num
        if self.num_Baum_iters > 0:
            nf = int(1.5 * self.num)
        responses, LAFs, oct_, lvl = self._detect(nf, self.mrSize)
        if self.num_Baum_iters > 0:
            responses, LAFs, oct_, lvl = self.getAffineShape(responses, LAFs, oct_, lvl, self.num)
        if do_ori:
            LAFs = self.getOrientation(LAFs, oct_, lvl)
        return denormalizeLAFs(LAFs, x.size(3), x.size(2)), responses
