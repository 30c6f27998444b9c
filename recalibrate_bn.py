"""python recalibrate_bn.py --trainer gan|segmenter --checkpoint IN.npz --out OUT.npz (--volumes PAIRS | --records LIST)
[--batches 200] [--batch-size 8] [--scope dam|all] [--seed S] -- re-estimate a checkpoint's batch-norm moving statistics as exact
population statistics over many slices (bnstats.py): PreciseBN on source slices, AdaBN on target-domain slices.  OUT.npz holds
every graph variable, the recalibrated statistics replaced, and pnp/global_step; every checkpoint consumer (restore,
test_native, evaluate_native.py, the ensembles) reads it as it reads the others."""
from pnp_b200.bnstats import main

if __name__ == "__main__":
    main()
