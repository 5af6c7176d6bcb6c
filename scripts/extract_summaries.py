"""One scalar of a TensorBoard log as a CSV: the reference's `extract_tensorboard.py` without tensorflow.

  python scripts/extract_summaries.py --log-dir DIR --scalar-name TAG

reads the event file `DIR/events.out.tfevents.*` (the first by name when there are several, as the reference takes the
first it lists) and writes `DIR/TAG.csv` with the columns wall_time, step, value, one row per event in file order.
TAG is e.g. train_reward, test_reward, loss/fplstm_0a_value_loss or train/dqn_0a_q; a tag with '/' goes into the
matching subdirectory of DIR, as in the reference.  Exits with status 1 when DIR holds no event file.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--log-dir", required=True, help="dir of tensorboard logs")
    p.add_argument("--scalar-name", default="train_reward", help="scalar names to be extraced")
    return p.parse_args(argv)


def main(argv=None):
    import pandas as pd
    from deeprl_signal_control_b200.agents.summary import event_files, read_scalars
    a = parse_args(argv)
    files = event_files(a.log_dir)
    if not files:
        print("no events.out.tfevents.* file in %s" % a.log_dir, file=sys.stderr)
        raise SystemExit(1)
    rows = read_scalars(files[0]).get(a.scalar_name, [])
    df = pd.DataFrame({"wall_time": [r[0] for r in rows], "step": [r[1] for r in rows],
                       "value": [r[2] for r in rows]})
    out = os.path.join(a.log_dir, a.scalar_name + ".csv")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    df.to_csv(out)
    return out


if __name__ == "__main__":
    main()
