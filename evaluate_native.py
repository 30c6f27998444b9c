"""python evaluate_native.py --trainer gan|segmenter --checkpoint CKPT.npz --pairs LIST --out DIR [--batch-size B]
[--hd-percentile Q] -- segment raw MMWHS subjects on their own voxel grid and score them there in mm (native.py):
DIR/native_pred/<name>_label.nii.gz and DIR/native.csv (with <organ>_hd<Q>_mm columns when Q is given, e.g. hd95_mm)."""
from pnp_b200.native import main

if __name__ == "__main__":
    main()
