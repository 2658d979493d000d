from .datasets import CSDataSet, CSDataLoader, CSDataTestSet, DeviceAugment, DeviceTestPreprocess, draw_augmentation, Augmentation  # noqa: F401
from .datasets import cityscapes_id_tables  # noqa: F401
from .datasets import VOCDataSet, VOCDataTestSet, numpy_mean, CS_SCALES, VOC_SCALES  # noqa: F401
from .datasets import CamVidDataSet, CAMVID_CLASSES, camvid_label_table, class_frequency_weights  # noqa: F401
