"""python prepare_data.py --modality ct|mr --pairs LIST --split train|val|test --out DIR ... -- the data preparation of the
reference's README step 1 (crop, intensity cut, z-score, augmented coronal slices), resampled on the GPU."""
from pnp_b200.prepare_data import main

if __name__ == "__main__":
    main()
