"""Sequential recommenders on the time-ordered samplers: FPMC and TransRec (high_order = 1)."""
