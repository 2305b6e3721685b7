"""Drop-in for reference `dataloader/train_loader.py` `FileLoader`, validation mode only.

Each file is a `.npy` patch as written by the reference's extract_patches.py: [H,W,4] (RGB, instance map) or
[H,W,5] (RGB, instance map, type map).  In "valid" mode the reference applies no augmentation, only a centre crop
of image and labels to `input_shape`; the targets come from `target_gen` on the cropped instance map and the type
map is cropped to `mask_shape`.  "train" mode needs the reference's augmentation pipeline, which is out of scope."""
import numpy as np

from ..models.hovernet.targets import cropping_center


class FileLoader(object):
    def __init__(self, file_list, with_type=False, input_shape=None, mask_shape=None, mode="train",
                 setup_augmentor=True, target_gen=None):
        assert input_shape is not None and mask_shape is not None
        if mode != "valid":
            raise NotImplementedError("FileLoader supports mode='valid' only (training augmentation is not provided)")
        self.mode = mode
        self.info_list = file_list
        self.with_type = with_type
        self.mask_shape = mask_shape
        self.input_shape = input_shape
        self.id = 0
        self.target_gen_func = target_gen[0]
        self.target_gen_kwargs = target_gen[1]

    def setup_augmentor(self, worker_id, seed):
        self.id = self.id + worker_id

    def __len__(self):
        return len(self.info_list)

    def load(self, idx):
        """(img uint8 [h,w,3], inst int32 [h,w], type int32 [h,w] or None), centre-cropped to input_shape."""
        data = np.load(self.info_list[idx])
        img = cropping_center(data[..., :3].astype("uint8"), self.input_shape)
        ann = cropping_center(data[..., 3:].astype("int32"), self.input_shape)
        return img, ann[..., 0], (ann[..., 1] if self.with_type else None)

    def __getitem__(self, idx):
        img, inst_map, type_map = self.load(idx)
        feed_dict = {"img": img}
        if self.with_type:
            feed_dict["tp_map"] = cropping_center(type_map.copy(), self.mask_shape)
        feed_dict.update(self.target_gen_func(inst_map, self.mask_shape, **self.target_gen_kwargs))
        return feed_dict
