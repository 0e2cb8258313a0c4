"""H100-native Balanced Group Softmax (BAGS) RoI classification head."""
__version__ = '0.1.0'
