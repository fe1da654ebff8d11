"""Drop-in for the reference's ``pi3`` package (VSLAM/thirdparty/Pi3/pi3): the model class under its module path."""
