"""Mirror of the reference's dotted paths for the hot-path plugins: replacing the `sgm.` prefix of a `target:`
in scripts/pub/configs/V3D_512.yaml by `v3d_b200.sgm.` selects the H100-native implementation
(INTEGRATION.md).  Only the classes on the path (SURVEY.md §8) exist here."""
