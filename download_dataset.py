#!/usr/bin/env python
"""Dataset preparation.  Parity with the reference's ``download_dataset.py`` (:1-29):
fetch MNIST-784 from OpenML, scale to [0,1], subtract the global mean, one-hot the labels,
85/15 split with seed 42, write ``x_{train,val}.parquet`` + ``y_{train,val}.npy``.

The GPU machines may have no network: ``--synthetic`` (or a failed download) writes
the deterministic MNIST-shaped synthetic set in the SAME file format instead, so train.py
and the unmodified reference can both consume it.  Files go to ``data/mnist_784/`` - the
directory train.py reads (the reference writes to ``../data`` and reads ``data``: a quirk
we do not copy)."""
import argparse
from pathlib import Path

import numpy as np


def download_MNIST(save_dir: Path):
    import pandas as pd
    from sklearn.datasets import fetch_openml
    from sklearn.model_selection import train_test_split

    x, y = fetch_openml("mnist_784", version=1, data_home="data_cache", return_X_y=True, as_frame=True)
    x = x.astype(np.float32) / 255.0
    x -= x.to_numpy().mean()
    y = pd.get_dummies(y).to_numpy().astype(np.float32)
    x_train, x_val, y_train, y_val = train_test_split(x, y, test_size=0.15, random_state=42)
    save_dir.mkdir(parents=True, exist_ok=True)
    x_train.to_parquet(save_dir / "x_train.parquet")
    x_val.to_parquet(save_dir / "x_val.parquet")
    np.save(save_dir / "y_train.npy", y_train)
    np.save(save_dir / "y_val.npy", y_val)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--save-dir", default="data/mnist_784/")
    ap.add_argument("--synthetic", action="store_true", help="skip the download, write synthetic MNIST-shaped data")
    args = ap.parse_args()
    save_dir = Path(args.save_dir)
    ok = False
    if not args.synthetic:
        try:
            download_MNIST(save_dir)
            ok = True
        except Exception as e:  # no network / OpenML unreachable
            print(f"download failed ({type(e).__name__}: {e}); falling back to synthetic data")
    if not ok:
        from shallowspeed_b200.dataset import write_reference_files

        write_reference_files(save_dir, overwrite=True)
    print("dataset written to", save_dir)
