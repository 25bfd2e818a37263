"""General recommenders of the MF family on the sm_90a hot path: MF (BPRMF / pointwise),
MLP, NeuMF, LightGCN, NGCF, APR, SpectralCF, WRMF, FISM (item similarity over the train history), and ItemKNN (the item-item neighbourhood baseline).  Resolved by name from main.py like the reference (main.py:30-40)."""
