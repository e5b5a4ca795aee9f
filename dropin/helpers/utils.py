"""`helpers.utils` as the reference scripts import it (helpers/utils.py).  The label table is read at import time
from metadata/class_labels_indices.csv relative to the CWD, exactly like the reference (helpers/utils.py:38)."""
from efficientat_b200.helpers.utils import (NAME_TO_WIDTH, exp_rampup, exp_warmup_linear_down,  # noqa: F401
                                            linear_rampdown, load_labels, mixstyle, mixup)

labels, ids = load_labels()
classes_num = len(labels)
