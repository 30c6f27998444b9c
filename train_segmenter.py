"""python train_segmenter.py ... -- same entry point as the reference's train_segmenter.py, H100-native underneath."""
from pnp_b200.train_segmenter import main

if __name__ == "__main__":
    main()
