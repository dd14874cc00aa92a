"""CPU: ops.cluster_head_loss and ops.multiclass_nms_groups refuse, with SSTB200Error and before any kernel runs, every input their
kernels would read as a raw device array but cannot: labels that are not int64 [M], bbox_targets that are not float32 [M, 8], num_pos
and avg factors that are not [T], a prediction of the wrong shape, and host tensors.  Shapes and dtypes are checked before devices, so
each misuse is named on a machine without a GPU; tests/test_gpu_cluster_head.py checks the device mismatches."""
import pytest
import torch

from sst_b200 import _lib, ops

M, T = 12, 2


def _args(**kw):
    a = dict(cls_logits=[torch.zeros(M, 1), torch.zeros(M, 3)], reg_preds=[torch.zeros(M, 8), torch.zeros(M, 8)],
             labels=[torch.zeros(M, dtype=torch.long), torch.zeros(M, dtype=torch.long)], bbox_targets=[torch.zeros(M, 8), torch.zeros(M, 8)],
             num_pos=torch.zeros(T, dtype=torch.long), cls_avg_factor=torch.ones(T), reg_avg_factor=torch.ones(T))
    a.update(kw)
    return a


CASES = {
    "labels int32": (dict(labels=[torch.zeros(M, dtype=torch.int32), torch.zeros(M, dtype=torch.long)]), "labels\\[0\\] must be int64"),
    "labels short": (dict(labels=[torch.zeros(M, dtype=torch.long), torch.zeros(M - 1, dtype=torch.long)]), "labels\\[1\\] must be int64"),
    "targets [M, 7]": (dict(bbox_targets=[torch.zeros(M, 7), torch.zeros(M, 8)]), "bbox_targets\\[0\\] must be float32"),
    "targets float64": (dict(bbox_targets=[torch.zeros(M, 8), torch.zeros(M, 8, dtype=torch.float64)]), "bbox_targets\\[1\\] must be float32"),
    "num_pos int32": (dict(num_pos=torch.zeros(T, dtype=torch.int32)), "num_pos must be int64"),
    "num_pos [T + 1]": (dict(num_pos=torch.zeros(T + 1, dtype=torch.long)), "num_pos must be int64"),
    "reg factor [1]": (dict(reg_avg_factor=torch.ones(1)), "reg_avg_factor must be float32"),
    "reg_preds [M, 7]": (dict(reg_preds=[torch.zeros(M, 8), torch.zeros(M, 7)]), "task 1"),
    "logits rows": (dict(cls_logits=[torch.zeros(M, 1), torch.zeros(M + 1, 3)]), "task 1"),
    "host tensors": ({}, "CUDA tensor"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_loss_refuses_misuse(case):
    kw, msg = CASES[case]
    with pytest.raises(_lib.SSTB200Error, match=msg):
        ops.cluster_head_loss(**_args(**kw), cfg=ops.ClusterHeadLossConfig())


def test_loss_refuses_task_count_mismatch():
    with pytest.raises(_lib.SSTB200Error, match="per task"):
        ops.cluster_head_loss(**_args(labels=[torch.zeros(M, dtype=torch.long)]), cfg=ops.ClusterHeadLossConfig())


def test_multiclass_nms_groups_refuses_host_tensors():
    boxes = torch.zeros(4, 7)
    z = torch.zeros(4, dtype=torch.long)
    with pytest.raises(_lib.SSTB200Error, match="CUDA"):
        ops.multiclass_nms_groups(boxes, torch.zeros(4, 5), z, z, torch.ones(4), z, 1, 1, [0.5], 10, True)
