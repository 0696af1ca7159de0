"""networks/tester.py (`render_test`) and the test-time metrics of networks/evaluator.py on the native kernels.

    render_test(position_embedder, view_embedder, model_coarse, model_fine, render_poses, hwk, args, gt_imgs=None, gt_labels=None,
                ins_rgbs=None, savedir=None, matched_file=None, crop_mask=None)                          tester.py:17-162
    psnr(rgb, gt), ssim(rgb, gt)            skimage 0.18.3 peak_signal_noise_ratio / structural_similarity(multichannel=True),
                                            data_range=1                                               tester.py:89-90
    ins_eval(pred_ins, gt_ins, gt_ins_num, ins_num, mask=None) -> (pred_label, ap_list, return_labels)  evaluator.py:125-175
    calculate_ap(IoUs_Metrics, gt_number, confidence=None, function_select='integral')                evaluator.py:77-122
    write_png(path, array)                  8-bit grey, RGB or RGBA PNG (zlib + struct; no imageio / cv2 / PIL)

Every metric is computed on the device by csrc/metrics.cu: PSNR, SSIM, the predicted labels, the joint histogram of predicted and
gt labels, per-label median confidences, the cost matrices, the assignment (the device LSAP solver of the training loss) and
the APs.  One small result struct is read back per frame.  The functions take CUDA tensors and raise RuntimeError on CPU tensors.
Rules and deviations from the original: DESIGN.md, "Evaluation metrics".

LPIPS: when the `lpips` package is importable and its model can be built, render_test computes it exactly as the original does
(VGG, inputs in [0, 1], on the device).  `lpips.LPIPS(net="vgg")` ships only its linear calibration layers; the VGG16 backbone
comes from torchvision's pretrained-weight download (or its local cache), which this project does not fetch.  Without the
package, or when the model cannot be built (for example no cached VGG16 weights and no network), the LPIPS column is NaN and one
warning says why."""
import ctypes as C
import json
import os
import struct
import warnings
import zlib

import numpy as np
import torch

from . import _lib
from .engine import get_context

_MAX_LABEL = 1 << 16                  # dmnerf_ins_label_rows ranks labels in [0, 65536)
_RANK_SLOTS = 128                     # distinct labels it ranks at most (ins_num + 1 <= 128)
_workspaces = {}


def _workspace(dev, n, k, H, W):
    ctx = get_context(dev)
    need = int(ctx.lib.dmnerf_eval_workspace_bytes(int(n), int(k), int(H), int(W)))
    ws = _workspaces.get(dev)
    if ws is None or ws.numel() < need:
        ws = torch.empty(max(need, 1), device=dev, dtype=torch.uint8)
        _workspaces[dev] = ws
    return ws


def _result_buffer(dev):
    return torch.zeros(C.sizeof(_lib.EvalResult), device=dev, dtype=torch.uint8)


def _read_result(buf):
    return _lib.EvalResult.from_buffer_copy(buf.cpu().numpy().tobytes())          # the one device -> host read


def _image_into(rgb, gt, res):
    if rgb.dim() != 3 or rgb.shape[-1] != 3 or tuple(rgb.shape) != tuple(gt.shape):
        raise ValueError("psnr / ssim: expected two [H, W, 3] images, got %s and %s" % (tuple(rgb.shape), tuple(gt.shape)))
    H, W = int(rgb.shape[0]), int(rgb.shape[1])
    if H < 7 or W < 7:
        raise ValueError("win_size exceeds image extent: %dx%d frame, 7x7 window (skimage structural_similarity)" % (H, W))
    rgb, gt = rgb.detach().contiguous().float(), gt.detach().to(rgb.device).contiguous().float()
    ctx = get_context(rgb.device)
    ws = _workspace(rgb.device, 0, 0, H, W)
    ctx.call("dmnerf_eval_image", _lib.ptr(rgb), _lib.ptr(gt), H, W, _lib.ptr(ws, torch.uint8), _lib.ptr(res, torch.uint8))


def image_metrics(rgb, gt):
    """(psnr, ssim) of two [H, W, 3] CUDA images with data_range 1, one read-back."""
    _lib.need_cuda("image_metrics", rgb, gt)
    res = _result_buffer(rgb.device)
    _image_into(rgb, gt, res)
    r = _read_result(res)
    return float(r.psnr), float(r.ssim)


def psnr(rgb, gt):
    """skimage.metrics.peak_signal_noise_ratio(rgb, gt, data_range=1) (scikit-image 0.18.3); a zero error gives inf."""
    return image_metrics(rgb, gt)[0]


def ssim(rgb, gt):
    """skimage.metrics.structural_similarity(rgb, gt, multichannel=True, data_range=1) (scikit-image 0.18.3)."""
    return image_metrics(rgb, gt)[1]


def _ins_eval_rows(ins, gt_row, gt_num, res, mask=None, mask_labels=None, mask_below=0):
    """Device ins_eval on ins [n, k] and gt ranks gt_row [n] int32 -> pred_label [n] int64 (device); the rest goes to `res`."""
    n, k = ins.shape
    dev = ins.device
    ctx = get_context(dev)
    ws = _workspace(dev, n, k, 0, 0)
    pred_label = torch.empty(n, device=dev, dtype=torch.int64)
    i32 = torch.int32
    ctx.call("dmnerf_ins_eval", _lib.ptr(ins), n, k, _lib.ptr(gt_row, i32), int(gt_num), _lib.ptr(mask), _lib.ptr(mask_labels, i32),
             int(mask_below), _lib.ptr(pred_label, torch.int64), _lib.ptr(ws, torch.uint8), _lib.ptr(res, torch.uint8))
    return pred_label


def _check_status(r):
    if r.status == 1:
        raise RuntimeError("ins_eval: the instance map holds NaN")
    if r.status != 0:
        raise RuntimeError("ins_eval: the assignment left a gt object unmatched (status %d)" % r.status)


def ins_eval(pred_ins, gt_ins, gt_ins_num, ins_num, mask=None):
    """evaluator.py:125-175.  pred_ins, gt_ins [..., ins_num] (gt_ins one-hot in its first gt_ins_num columns), mask [...] (0 =
    masked, the crop path).  Returns (pred_label [...] int64 CUDA tensor, ap_list (6 floats), return_labels int64 numpy array:
    the matched predicted label per gt object, or -1)."""
    _lib.need_cuda("ins_eval", pred_ins, gt_ins, mask)
    if pred_ins.shape[-1] != ins_num or tuple(gt_ins.shape) != tuple(pred_ins.shape):
        raise ValueError("ins_eval: pred_ins %s / gt_ins %s / ins_num %d are inconsistent"
                         % (tuple(pred_ins.shape), tuple(gt_ins.shape), ins_num))
    lead = tuple(pred_ins.shape[:-1])
    ins = pred_ins.detach().reshape(-1, ins_num).contiguous().float()
    gt = gt_ins.detach().reshape(-1, ins_num).contiguous().float()
    n = ins.shape[0]
    dev = ins.device
    ctx = get_context(dev)
    gt_row = torch.empty(n, device=dev, dtype=torch.int32)
    ctx.call("dmnerf_ins_dense_rows", _lib.ptr(gt), n, ins_num, int(gt_ins_num), _lib.ptr(gt_row, torch.int32))
    m = None if mask is None else mask.detach().reshape(-1).contiguous().float()
    res = _result_buffer(dev)
    pred_label = _ins_eval_rows(ins, gt_row, gt_ins_num, res, mask=m)
    r = _read_result(res)
    _check_status(r)
    return pred_label.reshape(lead), [float(v) for v in r.ap], np.array(r.return_labels[:int(gt_ins_num)], dtype=np.int64)


def calculate_ap(IoUs_Metrics, gt_number, confidence=None, function_select='integral'):
    """evaluator.py:77-122 (integral method only).  Matches are ordered by confidence, descending, ties in index order."""
    if function_select != 'integral':
        raise NotImplementedError("calculate_ap: only function_select='integral' (the one ins_eval uses) is implemented")
    _lib.need_cuda("calculate_ap", IoUs_Metrics, confidence)
    iou = IoUs_Metrics.detach().reshape(-1).contiguous().float()
    conf = None if confidence is None else confidence.detach().to(iou.device).reshape(-1).contiguous().float()
    ap = torch.empty(6, device=iou.device, dtype=torch.float32)
    ctx = get_context(iou.device)
    ctx.call("dmnerf_calculate_ap", _lib.ptr(iou), _lib.ptr(conf), iou.numel(), int(gt_number), _lib.ptr(ap))
    return [float(v) for v in ap.cpu()]


# ----------------------------------------------------------------------------------------------------------------- images
def write_png(path, img):
    """8-bit PNG of a uint8 array [H, W] (grey), [H, W, 3] (RGB) or [H, W, 4] (RGBA, straight alpha), no filtering, zlib
    level 6."""
    a = np.ascontiguousarray(np.asarray(img))
    if a.dtype != np.uint8 or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] not in (3, 4)):
        raise ValueError("write_png: expected uint8 [H, W], [H, W, 3] or [H, W, 4], got %s %s" % (a.dtype, a.shape))
    h, w = a.shape[:2]
    rows = a.reshape(h, -1)
    raw = np.concatenate([np.zeros((h, 1), np.uint8), rows], axis=1).tobytes()       # filter byte 0 per scanline

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

    color_type = 0 if a.ndim == 2 else (2 if a.shape[2] == 3 else 6)                 # grey, RGB, RGBA
    ihdr = struct.pack(">IIBBBBB", w, h, 8, color_type, 0, 0, 0)
    with open(path, "wb") as fh:
        fh.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", ihdr) + chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def _rgb_u8(rgb):
    return np.asarray(np.asarray(rgb, dtype=np.float64).reshape(3), dtype=np.float64).astype(np.uint8)


def colorize(labels, lut):
    """Device gather: out [..., 3] uint8 = lut[label] (lut [L, 3] uint8), black for labels outside [0, L)."""
    _lib.need_cuda("colorize", labels)
    lab = labels.contiguous()
    if lab.dtype not in (torch.int64, torch.int32):
        lab = lab.to(torch.int64)
    lut_d = torch.as_tensor(np.ascontiguousarray(lut, dtype=np.uint8).reshape(-1, 3)).to(lab.device)
    out = torch.empty(tuple(lab.shape) + (3,), device=lab.device, dtype=torch.uint8)
    ctx = get_context(lab.device)
    ctx.call("dmnerf_label_colors", _lib.ptr(lab, lab.dtype), int(lab.dtype == torch.int64), lab.numel(), _lib.ptr(lut_d, torch.uint8),
             lut_d.shape[0], _lib.ptr(out, torch.uint8))
    return out


def pred_label_lut(ins_map, ins_rgbs, color_dict, n_labels):
    """render_label2img (tools/visualizer.py:73-86) as a table: predicted label -> rgbs[color_dict[ins_map[label]]]."""
    lut = np.zeros((n_labels, 3), np.uint8)
    for key, gt_label in ins_map.items():
        if 0 <= int(key) < n_labels:
            lut[int(key)] = _rgb_u8(ins_rgbs[color_dict[str(gt_label)]])
    return lut


def gt_label_lut(ins_rgbs, color_dict, n_labels):
    """render_gt_label2img (tools/visualizer.py:57-69) as a table: label -> rgbs[color_dict[label]], black if not a key."""
    lut = np.zeros((n_labels, 3), np.uint8)
    for key, idx in color_dict.items():
        try:
            lab = int(key)
        except ValueError:
            continue
        if 0 <= lab < n_labels:
            lut[lab] = _rgb_u8(ins_rgbs[idx])
    return lut


# ----------------------------------------------------------------------------------------------------------------- render_test
_lpips_warned = False


def _lpips_model(device):
    """lpips.LPIPS(net="vgg") on `device`, or None (with one warning) when the package is missing or the model cannot be built."""
    global _lpips_warned
    try:
        import lpips
    except ImportError:
        why = "the lpips package is not installed"
    else:
        try:
            return lpips.LPIPS(net="vgg").to(device)
        except Exception as e:         # VGG16 weights missing from torchvision's cache with no network, or a broken install
            why = "lpips.LPIPS(net='vgg') could not be built (%s: %s)" % (type(e).__name__, e)
    if not _lpips_warned:
        warnings.warn("render_test: %s; the LPIPS column is NaN" % why)
        _lpips_warned = True
    return None


def _render_frame_device(H, W, K, c2w, position_embedder, view_embedder, model_coarse, model_fine, args, dev):
    """tester.py:57-77 with the maps kept on the device: native get_rays_k + dm_nerf, args.N_test rays per call."""
    from .helpers import get_rays_k, z_val_sample
    from .render import dm_nerf
    # c2w: numpy array, CPU or CUDA tensor (train_*.py pass device-resident poses), like the original's torch.Tensor(c2w)
    rays_o, rays_d = get_rays_k(H, W, K, torch.as_tensor(c2w, dtype=torch.float32, device=dev))
    rays_o, rays_d = rays_o.reshape(-1, 3), rays_d.reshape(-1, 3)
    n = H * W
    z = z_val_sample(args.N_test, args.near, args.far, args.N_samples, device=dev)
    rgbs, inss = [], []
    with torch.no_grad():                          # inference path: the fused kernel, never the training autograd path
        for step in range(0, n, args.N_test):
            cnt = min(args.N_test, n - step)
            z_chunk = z if cnt == args.N_test else z_val_sample(cnt, args.near, args.far, args.N_samples, device=dev)
            out = dm_nerf(torch.stack([rays_o[step:step + cnt], rays_d[step:step + cnt]], 0), position_embedder, view_embedder,
                          model_coarse, model_fine, z_chunk, args)
            rgbs.append(out["rgb_fine"])
            inss.append(out["ins_fine"])
    if len(rgbs) == 1:
        return rgbs[0], inss[0]
    return torch.cat(rgbs, 0), torch.cat(inss, 0)


def _frame_metrics(who, i, rgb, gt_img, ins, labels, valid_gt, ins_num, lpips_vgg, gt_row, n_valid, mask_labels=None):
    """The per-frame metric block of render_test (tester.py:86-120) and manipulator_eval (manipulator.py:276-307), with their
    two printed lines.  rgb, gt_img [H, W, 3], ins [n, k] and labels [n] int32 on the device; valid_gt: the frame's gt object
    ids (CPU tensor); gt_row [n] int32 and n_valid [1] int32: scratch.  PSNR and SSIM (one dmnerf_eval_image), LPIPS (NaN when
    lpips_vgg is None) and ins_eval on the gt ranks of `labels`; mask_labels: the crop path's mask (labels >= ins_num masked).
    One read-back.  Returns (psnr, ssim, lpips, 6 APs, ins_map {predicted label: gt id}, pred_label [n] int64 on the device).
    A frame with no gt object gets AP 1.0, an empty map and pred_label -1."""
    n_px = ins.shape[0]
    dev = ins.device
    gt_num = int(valid_gt.numel())
    if gt_num > ins_num or valid_gt.numel() >= _RANK_SLOTS:
        raise ValueError("%s: frame %d has %d gt objects for ins_num %d" % (who, i, gt_num, ins_num))
    ctx = get_context(dev)
    res = _result_buffer(dev)
    _image_into(rgb, gt_img, res)
    lpips_i = float("nan")
    if lpips_vgg is not None:
        lpips_i = lpips_vgg(rgb.permute(2, 0, 1).unsqueeze(0), gt_img.permute(2, 0, 1).unsqueeze(0)).item()
    if gt_num > 0:
        i32 = torch.int32
        ctx.call("dmnerf_ins_label_rows", _lib.ptr(labels, i32), n_px, _RANK_SLOTS, _lib.ptr(gt_row, i32), _lib.ptr(n_valid, i32))
        pred_label = _ins_eval_rows(ins, gt_row, gt_num, res, mask_labels=mask_labels, mask_below=ins_num)
    r = _read_result(res)
    if gt_num > 0:
        _check_status(r)
        ap = [float(v) for v in r.ap]
        matched = list(r.return_labels[:gt_num])
    else:                                                                 # no gt object: AP 1.0, labels -1
        ap = [1.0] * 6
        matched = []
        pred_label = torch.full((n_px,), -1, device=dev, dtype=torch.int64)
    psnr_i, ssim_i = float(r.psnr), float(r.ssim)
    print(f"PSNR: {psnr_i} SSIM: {ssim_i} LPIPS: {lpips_i}")
    gt_np = valid_gt.numpy()
    ins_map = {}
    for idx, lab in enumerate(matched):
        if lab != -1:
            ins_map[str(lab)] = int(gt_np[idx])
    print(f"APs: {ap}")
    return psnr_i, ssim_i, lpips_i, ap, ins_map, pred_label


def render_test(position_embedder, view_embedder, model_coarse, model_fine, render_poses, hwk, args, gt_imgs=None, gt_labels=None,
                ins_rgbs=None, savedir=None, matched_file=None, crop_mask=None):
    """networks/tester.py render_test, same signature, printed lines and files in `savedir`:
    {i:03d}.png (rendered RGB), instance_{i:03d}.png and {i}_ins_gt.png (label colours with the channel order cv2.imwrite stores),
    {i}_ins_gt_mask.png (gt labels cast to uint8), matching_log.json and test_results.txt (PSNR SSIM LPIPS AP50..AP95 per frame
    and the mean row).  Reads ./data/color_dict.json like the original.  With gt_imgs=None only the RGB images are written."""
    data_info = args.datadir.split('/')
    dataset_name, scene_name = data_info[2], data_info[-1]
    H, W, K = hwk
    H, W = int(H), int(W)
    dev = torch.device(getattr(args, "device", None) or next(model_fine.parameters()).device)
    if dev.type != "cuda":
        raise RuntimeError("render_test: the models must be on a CUDA device (no CPU fallback)")
    ins_num = int(args.ins_num)
    crop_idx = None
    oh, ow = H, W
    if crop_mask is not None:
        cm = torch.as_tensor(np.asarray(crop_mask.cpu() if torch.is_tensor(crop_mask) else crop_mask)).reshape(-1)
        crop_idx = torch.nonzero(cm == 1).reshape(-1).to(dev)
        oh, ow = int(args.crop_height), int(args.crop_width)
        if crop_idx.numel() != oh * ow:
            raise ValueError("render_test: crop mask selects %d pixels, crop_height x crop_width = %d" % (crop_idx.numel(), oh * ow))
    n_px = oh * ow

    have_gt = gt_imgs is not None
    if have_gt:
        gt_img_dev = torch.as_tensor(gt_imgs).to(dev, torch.float32)
        lab_cpu = torch.as_tensor(gt_labels).cpu()
        if crop_idx is not None:
            gt_img_dev = gt_img_dev.reshape(gt_img_dev.shape[0], -1, 3)[:, crop_idx].reshape(-1, oh, ow, 3)
            lab_cpu = lab_cpu.reshape(lab_cpu.shape[0], -1)[:, crop_idx.cpu()].reshape(-1, oh, ow)
        gt_img_dev = gt_img_dev.contiguous()
        if lab_cpu.numel() and (int(lab_cpu.min()) < 0 or int(lab_cpu.max()) >= _MAX_LABEL):
            raise ValueError("render_test: gt labels must be integers in [0, %d)" % _MAX_LABEL)
        lab_dev = lab_cpu.to(torch.int32).to(dev).contiguous()
        lpips_vgg = _lpips_model(dev)
    if matched_file is not None and os.path.exists(matched_file):
        os.remove(matched_file)

    with open('./data/color_dict.json', 'r') as fh:
        color_dict = json.load(fh)[dataset_name][scene_name]
    full_map = {}
    psnrs, ssims, lpipses, aps = [], [], [], []
    gt_lut = None
    if have_gt and savedir is not None:
        gt_lut = gt_label_lut(ins_rgbs, color_dict, int(lab_cpu.max()) + 1 if lab_cpu.numel() else 1)[:, ::-1]   # cv2: BGR
    gt_row = torch.empty(n_px, device=dev, dtype=torch.int32)
    n_valid = torch.empty(1, device=dev, dtype=torch.int32)

    with torch.no_grad():
        for i, c2w in enumerate(render_poses):
            print('=' * 50, i, '=' * 50)
            rgb, ins = _render_frame_device(H, W, K, c2w, position_embedder, view_embedder, model_coarse, model_fine, args, dev)
            if crop_idx is not None:
                rgb, ins = rgb[crop_idx], ins[crop_idx]
            rgb = rgb.reshape(oh, ow, 3).contiguous()
            ins = ins.reshape(n_px, -1).contiguous()
            pred_label = None
            ins_map = {}
            if have_gt:
                gt_label = lab_cpu[i]
                valid_gt = torch.unique(gt_label)
                if crop_idx is not None:
                    valid_gt = valid_gt[:-1]                                          # tester.py:99
                psnr_i, ssim_i, lpips_i, ap, ins_map, pred_label = _frame_metrics(
                    "render_test", i, rgb, gt_img_dev[i], ins, lab_dev[i], valid_gt, ins_num, lpips_vgg, gt_row, n_valid,
                    mask_labels=lab_dev[i] if crop_idx is not None else None)
                psnrs.append(psnr_i)
                ssims.append(ssim_i)
                lpipses.append(lpips_i)
                full_map[i] = ins_map
                aps.append(ap)

            if savedir is not None:
                rgb8 = (255 * np.clip(rgb.cpu().numpy(), 0, 1)).astype(np.uint8)      # to8b
                write_png(os.path.join(savedir, '{:03d}.png'.format(i)), rgb8)
                if have_gt:
                    lut = pred_label_lut(ins_map, ins_rgbs, color_dict, ins_num + 1)[:, ::-1]
                    write_png(os.path.join(savedir, f"instance_{str(i).zfill(3)}.png"),
                              colorize(pred_label.reshape(oh, ow), lut).cpu().numpy())
                    write_png(os.path.join(savedir, f'{i}_ins_gt.png'), colorize(lab_dev[i], gt_lut).cpu().numpy())
                    write_png(os.path.join(savedir, f'{i}_ins_gt_mask.png'), np.array(gt_label.numpy(), dtype=np.uint8))

    if have_gt:
        if savedir is not None:
            with open(os.path.join(savedir, 'matching_log.json'), 'w') as f:
                json.dump(full_map, f)
        aps = np.array(aps)
        output = np.stack([psnrs, ssims, lpipses, aps[:, 0], aps[:, 1], aps[:, 2], aps[:, 3], aps[:, 4], aps[:, 5]])
        output = output.transpose([1, 0])
        out_ap = np.mean(aps, axis=0)
        mean_output = np.array([np.mean(psnrs), np.mean(ssims), np.mean(lpipses),
                                out_ap[0], out_ap[1], out_ap[2], out_ap[3], out_ap[4], out_ap[5]]).reshape([1, 9])
        output = np.concatenate([output, mean_output], 0)
        if savedir is not None:
            np.savetxt(fname=os.path.join(savedir, 'test_results.txt'), X=output, fmt='%.6f', delimiter=' ')
        print('=' * 49, 'Avg', '=' * 49)
        print('PSNR: {:.4f}, SSIM: {:.4f},  LPIPS: {:.4f} '.format(np.mean(psnrs), np.mean(ssims), np.mean(lpipses)))
        print('AP50: {:.4f}, AP75: {:.4f}, AP80: {:.4f}, AP85: {:.4f}, AP90: {:.4f}, AP95: {:.4f}'
              .format(out_ap[0], out_ap[1], out_ap[2], out_ap[3], out_ap[4], out_ap[5]))
