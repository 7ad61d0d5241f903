from .data import MinMaxScaler, QuantileTransformer, RobustScaler, StandardScaler

__all__ = ["StandardScaler", "MinMaxScaler", "RobustScaler", "QuantileTransformer"]
