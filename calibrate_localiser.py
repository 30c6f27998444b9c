"""python calibrate_localiser.py --pairs MR_PAIRS --out localiser.json -- calibrate the heart localiser (localise.py) from labelled
pairs of the source modality: the median whole-heart extent and the margins between the whole-heart box and the box of the four
predicted structures, per coronal axis in mm.  evaluate_native.py --locate localiser.json then segments scans without labels."""
from pnp_b200.localise import main

if __name__ == "__main__":
    main()
