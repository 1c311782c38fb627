"""The batches the reference's single-rank test loader forms (maskrcnn_benchmark/data/build.py:207-240,290,483-485).

The reference evaluates ``TEST.IMS_PER_BATCH`` images per step and pads each batch to its largest image (``BatchCollator`` ->
``to_image_list``).  With ``DATALOADER.ASPECT_RATIO_GROUPING`` (the default) a ``GroupedBatchSampler`` over a ``SequentialSampler``
puts portrait and landscape images in separate batches; without it a ``BatchSampler`` takes the images in order.  Because Swin
windows, DyConv borders and the GLIP fusion see the zero padding, a batched result depends on which images share a batch, so
reproducing the reference's batched numbers needs its batches.
"""
import bisect


def reference_test_batches(image_hw, ims_per_batch, aspect_grouping=True):
    """The dataset's original image sizes ``image_hw`` [(height, width)] in dataset order (``get_img_info``) -> the lists of dataset
    indices the reference's test loader yields, in order.

    Grouping: group = bisect_right([1], h / w) (portrait and square images, h / w >= 1, form group 1).  Each group's images are split,
    in order, into batches of ``ims_per_batch`` (the last may be shorter), and the batches are ordered by their first index."""
    ims_per_batch = int(ims_per_batch)
    if ims_per_batch < 1:
        raise ValueError(f"ims_per_batch must be >= 1, got {ims_per_batch}")
    n = len(image_hw)
    if not aspect_grouping:
        return [list(range(i, min(i + ims_per_batch, n))) for i in range(0, n, ims_per_batch)]
    groups = {}
    for i, (h, w) in enumerate(image_hw):
        groups.setdefault(bisect.bisect_right([1], float(h) / float(w)), []).append(i)
    batches = [idx[j:j + ims_per_batch] for g in sorted(groups) for idx in (groups[g],) for j in range(0, len(idx), ims_per_batch)]
    return sorted(batches, key=lambda b: b[0])
