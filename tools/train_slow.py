"""main.lua's training actions for the slow (accurate) architecture on KITTI: ``-a train_tr`` and ``-a train_all``.

    python tools/train_slow.py kitti slow -a train_tr -data_root /data            # 14 epochs, then test_te with the new net
    python tools/train_slow.py kitti2015 slow -a train_all -data_root /data -out out   # on nnz_tr + nnz_te, then submit

The command line of tools/train.py (main.lua's positional layout and option names, -gpu 1-based) for arch 'slow' only: the
network options are -l1 -fm -ks -l2 -nh2 -lr -bs -mom -true1 -false1 -false2 (no -m / -pow), the augmentation options and
the stereo method's overrides are as there.  The net goes to <data_root>/net/net_<dataset>_slow_<args>.t7.
-checkpoint_steps K, -stop_after S and -resume checkpoint and resume a run as in tools/train.py:

    while python tools/train_slow.py kitti slow -a train_tr -data_root /data -resume -stop_after 3000; [ $? -eq 75 ]; do :; done
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import train  # noqa: E402


def parse_args(argv=None):
    return train.parse_args(argv, arch="slow")


def main(argv=None):
    return train.main(argv, arch="slow")


if __name__ == "__main__":
    sys.exit(main())
