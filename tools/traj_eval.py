"""Score an estimated trajectory against a ground-truth one (an addition beyond the reference; DESIGN §25).

    python tools/traj_eval.py EST.txt GT.txt

Both files are in the KITTI odometry format (12 numbers of a camera-to-world [R | t] per line, as fuse_raw.py -poses track
writes poses.txt) with one line per frame, both starting at the same frame.  Prints one line: ate (the RMSE of the
translations in metres, without alignment), rpe_t and rpe_r (the mean consecutive-frame relative error, metres and
degrees), t_err (%) and r_err (deg/m) over the odometry devkit's 100 .. 800 m segments (NaN when the path is shorter),
and the segment count.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    ap = argparse.ArgumentParser(prog="traj_eval.py", description=__doc__.splitlines()[0])
    ap.add_argument("est")
    ap.add_argument("gt")
    args = ap.parse_args(argv)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import track

    try:
        est, gt = track.read_poses(args.est), track.read_poses(args.gt)
        m = track.trajectory_metrics(est, gt)
    except (OSError, ValueError) as e:
        raise SystemExit("traj_eval.py: %s" % e)
    print(track.metrics_line(os.path.basename(args.est), m))
    return 0


if __name__ == "__main__":
    sys.exit(main())
