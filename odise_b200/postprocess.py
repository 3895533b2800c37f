"""Device-side post-processing (SURVEY.md §8f-3): the tail of CategoryODISE.forward without a clip_head
(odise/modeling/meta_arch/odise.py:326-370) — bilinear mask upsample, MaskFormer.semantic_inference and
MaskFormer.panoptic_inference / instance_inference (maskformer_model.py:280-380) with no host round trips: the reference syncs ~4x per
query through `.item()`.  sem_seg_postprocess (crop to the un-padded image, bilinear resize to the requested output size;
sem_seg_postprocess_before_inference=True in every ODISE config) is folded into the samplers of the three kernels."""
import ctypes
import torch

from . import lib
from .lib import Planes


class PostProcessor:
    def __init__(self, device, num_classes, thing_ids, object_mask_threshold=0.0, overlap_threshold=0.8, nmma=3):
        self.dev = torch.device(device)
        self.K = num_classes
        nmma = 3 if nmma == 2 else nmma            # the semantic-inference GEMM (K = Q) keeps the bf16x3 planes in every mode
        self.nmma, self.lo = nmma, nmma == 3
        it = torch.zeros(num_classes, dtype=torch.uint8)
        it[list(thing_ids)] = 1
        self.is_thing = it.to(self.dev)
        self.obj_thr, self.ov_thr = float(object_mask_threshold), float(overlap_threshold)

    @torch.no_grad()
    def __call__(self, pred_logits, pred_masks, H, W, semantic=True, panoptic=True, instance=False, topk=100,
                 panoptic_on=True, instance_masks=True, padded_size=None, image_size=None):
        """pred_logits [B, Q, K+1], pred_masks [B, Q, h, w] (device fp32) ->
        dict(sem_seg [B, K, H, W], panoptic_seg int32 [B, H, W], seg_info int32 [B, Q, 3], n_segments int32 [B]);
        instance=True adds dict(instances=dict(scores, pred_classes, query_index, valid [B, topk], query_masks u8
        [B, Q, H, W])): instance i of image b has the binary mask query_masks[b, query_index[b, i]] and is kept by the
        reference's panoptic_on filter iff valid[b, i].
        (H, W): output size ("height"/"width" of the request).  padded_size / image_size: the padded network input and the
        un-padded image inside it (images.tensor.shape[-2:], images.image_sizes[i]; odise.py:326-347); omit both when
        (H, W) is the padded input size itself."""
        B, Q, K1 = pred_logits.shape
        assert K1 == self.K + 1
        hs, ws = pred_masks.shape[-2:]
        dev, L = self.dev, lib.load()
        geom = None
        if padded_size is not None or image_size is not None:
            ph, pw = padded_size if padded_size is not None else (H, W)
            ih, iw = image_size if image_size is not None else (ph, pw)
            if (ph, pw, ih, iw) != (H, W, H, W):
                geom = ctypes.byref(lib.PostprocessGeom(int(ph), int(pw), int(ih), int(iw)))
        Qp = (Q + 7) // 8 * 8
        probs_t = torch.zeros(B * self.K, Qp, dtype=torch.float32, device=dev) if semantic else None
        scores = torch.empty(B * Q, dtype=torch.float32, device=dev)
        labels = torch.empty(B * Q, dtype=torch.int32, device=dev)
        keep = torch.empty(B * Q, dtype=torch.int32, device=dev)
        cl = pred_logits.contiguous()
        probs = torch.empty(B * Q, K1, dtype=torch.float32, device=dev) if instance else None
        lib._launch("odise_query_scores_f32", cl, probs, probs_t, scores, labels, keep, B, Q, Qp, K1, self.obj_thr)
        out = {}
        pm = pred_masks.contiguous()
        # ONE resampling pass over the mask logits feeds all requested heads (odise_postprocess_fused_f32)
        sig = Planes.empty(B * H * W, Qp, dev, lo=self.lo, ld=Qp) if semantic else None
        pan = seg_info = nseg = pws = None
        if panoptic:
            pan = torch.empty(B, H, W, dtype=torch.int32, device=dev)
            seg_info = torch.zeros(B, Q, 3, dtype=torch.int32, device=dev)
            nseg = torch.empty(B, dtype=torch.int32, device=dev)
            pws = torch.empty(int(L.odise_panoptic_ws_bytes(B, Q, H, W)), dtype=torch.uint8, device=dev)
        i_sc = i_cl = i_q = i_ok = qm = iws = None
        if instance:
            i_sc = torch.empty(B, topk, dtype=torch.float32, device=dev)
            i_cl = torch.empty(B, topk, dtype=torch.int32, device=dev)
            i_q = torch.empty(B, topk, dtype=torch.int32, device=dev)
            i_ok = torch.empty(B, topk, dtype=torch.int32, device=dev)
            qm = torch.empty(B, Q, H, W, dtype=torch.uint8, device=dev) if instance_masks else None
            iws = torch.empty(int(L.odise_postprocess_fused_ws_bytes(B, Q, H, W)), dtype=torch.uint8, device=dev)
        if semantic or panoptic or instance:
            lib._launch("odise_postprocess_fused_f32", pm, sig.hi if sig else None, sig.lo if sig else None, Qp, scores,
                        labels, keep, self.is_thing, pan, seg_info, nseg, pws, self.ov_thr, probs, i_sc, i_cl, i_q, i_ok,
                        qm, iws, topk, 1 if panoptic_on else 0, B, Q, self.K, hs, ws, H, W, geom)
        if semantic:
            # sem[b] = P_b^T [K, Q] @ sig_b^T [Q, HW]: swapped-operand GEMM writes the reference's [K, H, W] layout
            ptp = lib.split(probs_t, lo=self.lo)
            sem = torch.empty(B, self.K, H * W, dtype=torch.float32, device=dev)
            lib.gemm(ptp, sig, M=self.K, N=H * W, K=Qp, nmma=self.nmma, batch=B, a_bs=self.K * ptp.ld, b_bs=H * W * sig.ld,
                     out=sem, ld_out=H * W, out_bs=self.K * H * W)
            out["sem_seg"] = sem.view(B, self.K, H, W)
        if panoptic:
            out.update(panoptic_seg=pan, seg_info=seg_info, n_segments=nseg)
        if instance:
            out["instances"] = dict(scores=i_sc, pred_classes=i_cl, query_index=i_q, valid=i_ok, query_masks=qm)
        out.update(scores=scores.view(B, Q), labels=labels.view(B, Q), keep=keep.view(B, Q))
        return out

    @staticmethod
    def segments_info(seg_info, n_segments):
        """host-side view (one D2H at the very end): list per image of dicts like the reference's."""
        si, ns = seg_info.cpu(), n_segments.cpu()
        return [[{"id": int(r[0]), "isthing": bool(r[1]), "category_id": int(r[2])} for r in si[b, :int(ns[b])]]
                for b in range(si.shape[0])]
