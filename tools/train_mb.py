"""main.lua's training actions on Middlebury for the fast and slow architectures: ``-a train_tr`` and ``-a train_all``.

    python tools/train_mb.py mb fast -a train_tr -data_root /data               # 14 epochs, then test_te with the new net
    python tools/train_mb.py mb slow -a train_all -rect perfect -data_root /data -out out   # nnz_tr + nnz_te, then submit

The command line of tools/train.py (main.lua's positional layout and option names, -gpu 1-based) for dataset mb: main.lua's
mb presets (-l1 5, fm 64 'fast' / 112 'slow', the Middlebury augmentation), plus -ds (stored, no effect, as in main.lua),
-d_exp, -d_light and -rect perfect|imperfect.  The set is <data_root>/data.mb.<rect>_gray, as tools/preprocess_mb.py writes
it; the net goes to <data_root>/net/net_mb_<arch>_<args>.t7.  Refused before any GPU work: kitti / kitti2015 (train.py,
train_slow.py), -color rgb, -subset < 1, -debug, each arch's foreign options, and a set the loader cannot use (see
mc-cnn_b200/train.py's MbTrainSet).  -checkpoint_steps K, -stop_after S and -resume checkpoint and resume a run as in
tools/train.py; the checkpoint also holds the words the light / exposure draws hand back to the stream:

    while python tools/train_mb.py mb fast -a train_tr -data_root /data -resume -stop_after 3000; [ $? -eq 75 ]; do :; done
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import train  # noqa: E402


def parse_args(argv=None):
    return train.parse_args(argv, arch=None)


def main(argv=None):
    return train.main(argv, arch=None)


if __name__ == "__main__":
    sys.exit(main())
