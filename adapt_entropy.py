"""python adapt_entropy.py --trainer gan|segmenter --checkpoint IN.npz --out OUT.npz (--volumes PAIRS | --records LIST)
[--steps 100] [--lr 1e-4] [--batch-size 8] [--recalibrate-batches 200] [--seed S] -- adapt a checkpoint to unlabelled slices by
test-time entropy minimisation of its batch-norm scales and shifts (TENT, tent.py), then re-estimate their moving statistics
over further slices.  OUT.npz holds every graph variable and pnp/global_step; every checkpoint consumer (restore, test_native,
evaluate_native.py, the ensembles) reads it as it reads the others.  <OUT stem>_entropy.csv logs the mean entropy and the mean
class probabilities of every step."""
from pnp_b200.tent import main

if __name__ == "__main__":
    main()
