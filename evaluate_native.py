"""python evaluate_native.py --trainer gan|segmenter --checkpoint CKPT.npz [CKPT2.npz ...] (--pairs LIST | --images LIST --locate
CAL.json) --out DIR [--batch-size B] [--locate CAL.json] [--hd-percentile Q] [--largest-component 6|26] [--tta-rotations DEG ...]
[--tta-scales S ...] -- segment raw MMWHS subjects on their own voxel grid and score them there in mm (native.py): DIR/native_pred/<name>_label.nii.gz and DIR/native.csv (with
<organ>_hd<Q>_mm columns when Q is given, e.g. hd95_mm).  Several checkpoints and / or test-time rotations and scales are
ensembled: their class probabilities are summed at every native voxel before the argmax (native.csv adds members and
<organ>_dice_first).  --locate crops each scan at the heart box the network itself locates (localise.py; CAL.json from
calibrate_localiser.py) instead of the ground-truth box: with --pairs the located crop is scored (native.csv adds windows,
iterations, converged, box_iou, box_err_mm), with --images (one unlabelled image path per line) nothing is scored and
DIR/located.csv lists the boxes and organ volumes."""
from pnp_b200.native import main

if __name__ == "__main__":
    main()
