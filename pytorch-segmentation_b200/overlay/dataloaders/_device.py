"""Device mode for the reference's CityScapes, VOC and ADE20K datasets.  The reference's loader classes build their
dataset by module-global name, so each reference file is also loaded privately and, in that private copy only, the
dataset name is bound to the device-mode subclass of the reference's own (public) class; the loaders here are the private
copies' classes.  The reference's modules `dataloaders.cityscapes` etc. stay untouched."""
import importlib
import importlib.util
import os
import random

import numpy as np
from PIL import Image

from seg_b200.data import DeviceSample, device_collate, draw_augmentation


def _reference(name):
    """(the reference's module, through the package's __path__; a private copy of the same file)"""
    public = importlib.import_module(f"{__package__}.{name}")
    spec = importlib.util.spec_from_file_location(f"_reference_dataloaders_{name}", public.__file__)
    private = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(private)
    return public, private


def device_data_enabled():
    """SEG_DEVICE_DATA=0 keeps every dataset on the reference's path (with OpenCV's IPP dispatch the reference's resized
    images differ from the device's by one level on under 1 % of the pixels, DESIGN.md §7)."""
    return os.environ.get("SEG_DEVICE_DATA", "1") != "0"


class DeviceMode:
    """Mixin for a reference dataset class.  `device_mode` is True when the kernels build the configuration: a crop_size,
    `augment` or `val`, no `return_id`, SEG_DEVICE_DATA not 0; otherwise __getitem__ is the reference's, unchanged."""

    LABEL_MAP = None  # 256-entry int32 table applied to the raw uint8 label, or None

    def _init_device_mode(self):
        self.device_mode = bool(device_data_enabled() and self.crop_size and (self.augment or self.val) and not self.return_id)
        self.label_map = None if self.LABEL_MAP is None else np.asarray(self.LABEL_MAP, dtype=np.int32)

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self._init_device_mode()

    def _load_raw(self, index):
        """(image uint8 [H,W,3], label [H,W]) as _load_data decodes them, before its float / int32 casts and its label
        remap.  Returns (image, label, label_map): a label that is not uint8 is remapped here and comes back as int32."""
        raise NotImplementedError

    def __getitem__(self, index):
        if not self.device_mode:
            return super().__getitem__(index)
        image, label, lmap = self._load_raw(index)
        if self.val:
            draws = None
        else:
            (h, w), angle, y0, x0, f, sigma = draw_augmentation(image.shape[0], image.shape[1], int(self.crop_size), self.base_size,
                                                               self.scale, self.rotate, self.flip, self.blur, random)
            draws = (h, w, angle, y0, x0, f, sigma)
        return DeviceSample(image, label, draws, int(self.crop_size), lmap)

    def _raw_label(self, label, host_map):
        if label.dtype == np.uint8:
            return label, self.label_map
        return np.ascontiguousarray(host_map(label.astype(np.int32)), dtype=np.int32), None


def _device_loader(ref_loader):
    """The private copy's loader class (its dataset is the device-mode subclass); in device mode the loader and
    get_val_loader() pack batches with device_collate in the workers."""

    class Loader(ref_loader):
        def __init__(self, *args, **kwargs):
            super().__init__(*args, **kwargs)
            if self.dataset.device_mode:
                self.collate_fn = device_collate
                self.init_kwargs["collate_fn"] = device_collate

    Loader.__name__ = Loader.__qualname__ = ref_loader.__name__
    return Loader


# ------------------------------------------------------------------ CityScapes
_cs, _cs_private = _reference("cityscapes")


def cityscapes_label_map():
    """cityscapes.py:53-54's ID_TO_TRAINID loop run once over the 256 uint8 values: each pixel's result depends only on its
    own value, so map[raw] equals the per-pixel loop's result for every pixel."""
    t = np.arange(256, dtype=np.int32)
    for k, v in _cs.ID_TO_TRAINID.items():
        t[t == k] = v
    return t


def _cityscapes_host_map(label):
    for k, v in _cs.ID_TO_TRAINID.items():
        label[label == k] = v
    return label


class CityScapesDataset(DeviceMode, _cs.CityScapesDataset):
    LABEL_MAP = cityscapes_label_map()

    def _load_raw(self, index):
        image_path, label_path = self.files[index]
        image = np.asarray(Image.open(image_path).convert('RGB'))
        label, lmap = self._raw_label(np.asarray(Image.open(label_path)), _cityscapes_host_map)
        return image, label, lmap


_cs_private.CityScapesDataset = CityScapesDataset
CityScapes = _device_loader(_cs_private.CityScapes)


# ------------------------------------------------------------------ VOC (no label map)
_voc, _voc_private = _reference("voc")


class _VOCRaw(DeviceMode):
    def _raw_image_label(self, image_path, label_path):
        image = np.asarray(Image.open(image_path))
        label, lmap = self._raw_label(np.asarray(Image.open(label_path)), lambda lab: lab)
        return image, label, lmap


class VOCDataset(_VOCRaw, _voc.VOCDataset):
    def _load_raw(self, index):
        image_id = self.files[index]
        return self._raw_image_label(os.path.join(self.image_dir, image_id + '.jpg'), os.path.join(self.label_dir, image_id + '.png'))


class VOCAugDataset(_VOCRaw, _voc.VOCAugDataset):
    def _load_raw(self, index):
        return self._raw_image_label(os.path.join(self.root, self.files[index][1:]), os.path.join(self.root, self.labels[index][1:]))


_voc_private.VOCDataset, _voc_private.VOCAugDataset = VOCDataset, VOCAugDataset
VOC = _device_loader(_voc_private.VOC)


# ------------------------------------------------------------------ ADE20K (v -> v - 1)
_ade, _ade_private = _reference("ade20k")


class ADE20KDataset(DeviceMode, _ade.ADE20KDataset):
    LABEL_MAP = np.arange(256, dtype=np.int32) - 1  # ade20k.py:30: "from -1 to 149"

    def _load_raw(self, index):
        image_id = self.files[index]
        image = np.asarray(Image.open(os.path.join(self.image_dir, image_id + '.jpg')).convert('RGB'))
        label, lmap = self._raw_label(np.asarray(Image.open(os.path.join(self.label_dir, image_id + '.png'))), lambda lab: lab - 1)
        return image, label, lmap


_ade_private.ADE20KDataset = ADE20KDataset
ADE20K = _device_loader(_ade_private.ADE20K)
