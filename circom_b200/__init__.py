"""circom_b200: Hopper-native witness generation and R1CS evaluation for circom circuits."""
__version__ = "0.1.0"
