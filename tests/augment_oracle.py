"""CPU oracle of the augmentation chain with EXPLICIT parameters, through cv2: what tool/train.py's train_transform
(util/transform.py) computes for one sample once its random draws are known (`semseg_b200.augment.AugParams`).
Test and benchmark infrastructure only: the product package never imports cv2."""
import cv2
import numpy as np
import torch


def augment_one(image, label, p, crop_h, crop_w, mean, std, ignore_label=255):
    """uint8 RGB HWC image and uint8 HW label -> (fp32 [3,ch,cw], int64 [ch,cw]) tensors for draws `p`."""
    image = np.float32(image)
    h, w = label.shape
    if p.fx != 1.0 or p.fy != 1.0:
        image = cv2.resize(image, None, fx=p.fx, fy=p.fy, interpolation=cv2.INTER_LINEAR)
        label = cv2.resize(label, None, fx=p.fx, fy=p.fy, interpolation=cv2.INTER_NEAREST)
    if p.angle is not None:
        h, w = label.shape
        matrix = cv2.getRotationMatrix2D((w / 2, h / 2), p.angle, 1)
        image = cv2.warpAffine(image, matrix, (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT,
                               borderValue=mean)
        label = cv2.warpAffine(label, matrix, (w, h), flags=cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT,
                               borderValue=ignore_label)
    if p.blur:
        image = cv2.GaussianBlur(image, (5, 5), 0)
    if p.flip:
        image = cv2.flip(image, 1)
        label = cv2.flip(label, 1)
    h, w = label.shape
    pad_h, pad_w = max(crop_h - h, 0), max(crop_w - w, 0)
    if pad_h > 0 or pad_w > 0:
        image = cv2.copyMakeBorder(image, pad_h // 2, pad_h - pad_h // 2, pad_w // 2, pad_w - pad_w // 2,
                                   cv2.BORDER_CONSTANT, value=mean)
        label = cv2.copyMakeBorder(label, pad_h // 2, pad_h - pad_h // 2, pad_w // 2, pad_w - pad_w // 2,
                                   cv2.BORDER_CONSTANT, value=ignore_label)
    image = image[p.h_off:p.h_off + crop_h, p.w_off:p.w_off + crop_w]
    label = label[p.h_off:p.h_off + crop_h, p.w_off:p.w_off + crop_w]
    t = torch.from_numpy(np.ascontiguousarray(image.transpose(2, 0, 1))).float()
    for c, m, s in zip(t, mean, std):
        c.sub_(m).div_(s)
    return t, torch.from_numpy(np.ascontiguousarray(label)).long()


def augment_batch(samples, params, crop_h, crop_w, mean, std, ignore_label=255):
    """[(image, label), ...] with one AugParams each -> (fp32 [N,3,ch,cw], int64 [N,ch,cw]) CPU tensors."""
    outs = [augment_one(i, l, p, crop_h, crop_w, mean, std, ignore_label) for (i, l), p in zip(samples, params)]
    return torch.stack([o[0] for o in outs]), torch.stack([o[1] for o in outs])
