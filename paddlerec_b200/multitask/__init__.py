"""Multi-task models: mirrors of the reference's models/multitask/<model>/ plugin directories."""
